// sm_90a copy kernels of the checkpoint data plane.
//
//   tsnap_bulk_copy_kernel : dense 16B-aligned runs.  One warp per CTA, one elected lane drives a
//       ring of shared-memory stages with the bulk async-copy engine (TMA, 1-D form):
//       cp.async.bulk global->shared (mbarrier complete_tx) then cp.async.bulk shared->global
//       (bulk_group).  No register staging, ~10 instructions per 16 KiB.
//   tsnap_lsu_copy_kernel  : everything else — dense runs at odd alignment (slab members sit back
//       to back with no padding, T:batcher.py:307), strided views (narrow on dim != 0, transposes,
//       reshard-on-load overlap boxes, T:io_preparers/sharded_tensor.py:285-298) and fused dtype
//       casts.  Destination-aligned 16 B stores, widest naturally aligned loads.
//   (transposes and short-run column shards the TMA unit can address: transpose_tma.cu)
//
// Both are persistent: grid = SMs x resident CTAs, tiles taken round-robin from a host-built tile
// table (plan.h).  HBM-bound byte movement: algorithmic traffic = 2 x payload bytes.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "convert.h"
#include "kernels.h"
#include "ptx.cuh"

namespace tsnap {

// ------------------------------------------------------------------------------------------------
// bulk (TMA) copy kernel
// ------------------------------------------------------------------------------------------------
// Piece = one <= kStageBytes slice of a tile.  A cursor walks this CTA's tiles and yields pieces in
// order; the same order is used for loads and stores, so stage = piece_ordinal % kStages.
struct PieceCursor {
    const Member* members;
    const Tile* tiles;
    uint32_t ntiles;
    uint32_t tile;       // current tile (global index)
    uint64_t pos, end;   // byte cursor inside the current member
    const char* src;
    char* dst;
    uint32_t stride;
    bool open;
};

__device__ __forceinline__ bool cursor_next(PieceCursor& c, uint32_t stage_bytes, const char** src, char** dst,
                                            uint32_t* bytes) {
    while (true) {
        if (c.open && c.pos < c.end) {
            uint64_t n = c.end - c.pos;
            if (n > stage_bytes) n = stage_bytes;
            *src = c.src + c.pos;
            *dst = c.dst + c.pos;
            *bytes = (uint32_t)n;
            c.pos += n;
            return true;
        }
        if (c.open) c.tile += c.stride;
        if (c.tile >= c.ntiles) return false;
        const Tile t = c.tiles[c.tile];
        const Member* m = c.members + t.member;
        c.src = reinterpret_cast<const char*>(m->src);
        c.dst = reinterpret_cast<char*>(m->dst);
        tile_range_bulk(*m, t.index, &c.pos, &c.end);
        c.open = true;
    }
}

template <int kStages, int kStageBytes>
__global__ void __launch_bounds__(32) tsnap_bulk_copy_kernel(const Member* __restrict__ members,
                                                             const Tile* __restrict__ tiles, uint32_t ntiles) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    // [kStages * kStageBytes data][kStages mbarriers]
    unsigned char* data = smem_raw;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + kStages * kStageBytes);
    if (threadIdx.x != 0) return;  // one elected lane drives the copy engine

    for (int s = 0; s < kStages; ++s) mbar_init(smem_u32(&bars[s]), 1);
    fence_mbar_init();
    fence_proxy_async_smem();
    const uint64_t policy = policy_evict_first();

    PieceCursor cur;
    cur.members = members;
    cur.tiles = tiles;
    cur.ntiles = ntiles;
    cur.tile = blockIdx.x;
    cur.stride = gridDim.x;
    cur.open = false;
    cur.pos = cur.end = 0;

    char* st_dst[kStages];
    uint32_t st_bytes[kStages];
    uint32_t issued = 0, stored = 0;

    const char* src;
    char* dst;
    uint32_t bytes;
    // prologue: fill the ring
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
        if (issued == (uint32_t)s && cursor_next(cur, kStageBytes, &src, &dst, &bytes)) {
            const uint32_t bar = smem_u32(&bars[s]);
            mbar_expect_tx(bar, bytes);
            bulk_g2s(smem_u32(data + s * kStageBytes), src, bytes, bar, policy);
            st_dst[s] = dst;
            st_bytes[s] = bytes;
            ++issued;
        }
    }
    while (stored < issued) {
        const uint32_t s = stored % kStages;
        mbar_wait(smem_u32(&bars[s]), (stored / kStages) & 1);
        // bytes landed through the async proxy and are read back by it; the fence orders the
        // mbarrier observation before the store is issued.
        fence_proxy_async_smem();
        char* d = nullptr;
        uint32_t b = 0;
#pragma unroll
        for (int k = 0; k < kStages; ++k)
            if (k == (int)s) {
                d = st_dst[k];
                b = st_bytes[k];
            }
        bulk_s2g(d, smem_u32(data + s * kStageBytes), b);
        bulk_commit();
        ++stored;
        // the stage written out one iteration ago is free once all but the newest store group
        // have finished reading shared memory
        if (stored >= 2) {
            bulk_wait_read<1>();
            if (cursor_next(cur, kStageBytes, &src, &dst, &bytes)) {
                const uint32_t fs = (stored - 2) % kStages;
                const uint32_t bar = smem_u32(&bars[fs]);
                mbar_expect_tx(bar, bytes);
                bulk_g2s(smem_u32(data + fs * kStageBytes), src, bytes, bar, policy);
#pragma unroll
                for (int k = 0; k < kStages; ++k)
                    if (k == (int)fs) {
                        st_dst[k] = dst;
                        st_bytes[k] = bytes;
                    }
                ++issued;
            }
        }
    }
    bulk_wait_all<0>();
}

// ------------------------------------------------------------------------------------------------
// rows kernel: strided members with long 16 B-aligned runs, run by run through the copy engine
// ------------------------------------------------------------------------------------------------
// Same ring as the dense kernel (kStages x kStageBytes of shared memory, mbarrier per stage, bulk async-groups
// for the stores), but warp-collective: a stage holds up to kStageBytes of the member's LOGICAL bytes — a
// sequence of run segments — and the 32 lanes issue the per-run cp.async.bulk requests in parallel.  A side
// whose runs are adjacent (the wire image on save, the file image on restore) is moved with ONE request per
// stage.  No data passes through registers (SASS: UBLKCP.S.G / UBLKCP.G.S only).
struct RowsPiece {
    uint32_t member;  // index into the member table
    uint64_t pos;     // logical byte position inside the member
    uint32_t n;       // logical bytes
};

struct RowsCursor {
    const Member* members;
    const Tile* tiles;
    uint32_t ntiles, tile, stride;
    uint64_t pos, end;
    uint32_t member;
    bool open;
};

__device__ __forceinline__ bool rows_next(RowsCursor& c, uint32_t stage_bytes, RowsPiece* out) {
    while (true) {
        if (c.open && c.pos < c.end) {
            uint64_t n = c.end - c.pos;
            if (n > stage_bytes) n = stage_bytes;
            out->member = c.member;
            out->pos = c.pos;
            out->n = (uint32_t)n;
            c.pos += n;
            return true;
        }
        if (c.open) c.tile += c.stride;
        if (c.tile >= c.ntiles) return false;
        const Tile t = c.tiles[c.tile];
        c.member = t.member;
        tile_range_bulk(c.members[t.member], t.index, &c.pos, &c.end);
        c.open = true;
    }
}

__device__ __forceinline__ void rows_offsets(const Member& m, uint64_t row, int64_t* so, int64_t* dofs) {
    if (m.nouter == 1) {
        *so = (int64_t)row * m.sstride[0];
        *dofs = (int64_t)row * m.dstride[0];
        return;
    }
    int64_t s = 0, d = 0;
    for (int i = (int)m.nouter - 1; i >= 0; --i) {
        const uint64_t sz = (uint64_t)m.osize[i];
        const uint64_t idx = row % sz;
        row /= sz;
        s += (int64_t)idx * m.sstride[i];
        d += (int64_t)idx * m.dstride[i];
    }
    *so = s;
    *dofs = d;
}

// issues the copy-engine requests of one piece on one side.  kLoad: global -> stage (completion on `bar`),
// else stage -> global (bulk async-group of the issuing lane).
template <bool kLoad>
__device__ __forceinline__ void rows_issue(const Member& m, uint64_t pos, uint32_t n, uint32_t stage_smem, uint32_t bar,
                                           uint64_t policy, uint32_t lane) {
    const bool dense = (m.shift & (kLoad ? kRowsSrcDense : kRowsDstDense)) != 0;
    if (dense) {
        if (lane == 0) {
            if (kLoad) bulk_g2s(stage_smem, reinterpret_cast<const char*>(m.src) + pos, n, bar, policy);
            else bulk_s2g(reinterpret_cast<char*>(m.dst) + pos, stage_smem, n);
        }
        return;
    }
    const uint64_t inner = m.inner;
    const uint64_t row0 = pos / inner;
    const uint64_t col0 = pos - row0 * inner;
    uint64_t len0 = inner - col0;
    if (len0 > n) len0 = n;
    const uint32_t nseg = 1 + (uint32_t)((n - len0 + inner - 1) / inner);
    for (uint32_t k = lane; k < nseg; k += 32) {
        const uint64_t seg_off = k == 0 ? 0 : len0 + (uint64_t)(k - 1) * inner;  // inside the stage
        uint64_t len = k == 0 ? len0 : inner;
        if (seg_off + len > n) len = n - seg_off;
        int64_t so, dofs;
        rows_offsets(m, row0 + k, &so, &dofs);
        const uint64_t col = k == 0 ? col0 : 0;
        if (kLoad) bulk_g2s(stage_smem + (uint32_t)seg_off, reinterpret_cast<const char*>(m.src) + so + col, (uint32_t)len, bar, policy);
        else bulk_s2g(reinterpret_cast<char*>(m.dst) + dofs + col, stage_smem + (uint32_t)seg_off, (uint32_t)len);
    }
}

template <int kStages, int kStageBytes>
__global__ void __launch_bounds__(32) tsnap_rows_copy_kernel(const Member* __restrict__ members,
                                                             const Tile* __restrict__ tiles, uint32_t ntiles) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    // [kStages * kStageBytes data][kStages member records][kStages mbarriers]
    unsigned char* data = smem_raw;
    Member* st_m = reinterpret_cast<Member*>(smem_raw + kStages * kStageBytes);
    uint64_t* bars = reinterpret_cast<uint64_t*>(st_m + kStages);
    const uint32_t lane = threadIdx.x;
    if (lane == 0) {
        for (int s = 0; s < kStages; ++s) mbar_init(smem_u32(&bars[s]), 1);
        fence_mbar_init();
        fence_proxy_async_smem();
    }
    __syncwarp();
    const uint64_t policy = policy_evict_first();

    RowsCursor cur;
    cur.members = members;
    cur.tiles = tiles;
    cur.ntiles = ntiles;
    cur.tile = blockIdx.x;
    cur.stride = gridDim.x;
    cur.open = false;
    cur.pos = cur.end = 0;
    cur.member = 0;

    uint64_t st_pos[kStages];
    uint32_t st_n[kStages];
    uint32_t issued = 0, stored = 0;

    // stage `s` <- piece `p`: the member record travels with the stage (loads of the next member are in flight while
    // the previous member's stage is being stored)
    auto load_piece = [&](int s, const RowsPiece& p) {
        const uint32_t* g = reinterpret_cast<const uint32_t*>(members + p.member);
        uint32_t* d = reinterpret_cast<uint32_t*>(&st_m[s]);
        for (uint32_t i = lane; i < sizeof(Member) / 4; i += 32) d[i] = g[i];
        const uint32_t bar = smem_u32(&bars[s]);
        if (lane == 0) mbar_expect_tx(bar, p.n);
        __syncwarp();
        rows_issue<true>(st_m[s], p.pos, p.n, smem_u32(data + s * kStageBytes), bar, policy, lane);
    };

    RowsPiece p;
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
        if (issued == (uint32_t)s && rows_next(cur, kStageBytes, &p)) {
            load_piece(s, p);
            st_pos[s] = p.pos;
            st_n[s] = p.n;
            ++issued;
        }
    }
    while (stored < issued) {
        const uint32_t s = stored % kStages;
        mbar_wait(smem_u32(&bars[s]), (stored / kStages) & 1);
        fence_proxy_async_smem();
        uint64_t pos = 0;
        uint32_t n = 0;
#pragma unroll
        for (int k = 0; k < kStages; ++k)
            if (k == (int)s) {
                pos = st_pos[k];
                n = st_n[k];
            }
        rows_issue<false>(st_m[s], pos, n, smem_u32(data + s * kStageBytes), 0, policy, lane);
        bulk_commit();
        ++stored;
        if (stored >= 2) {
            bulk_wait_read<1>();  // every lane: all but its newest store group have finished reading shared memory
            __syncwarp();
            if (rows_next(cur, kStageBytes, &p)) {
                const uint32_t fs = (stored - 2) % kStages;
                load_piece((int)fs, p);
#pragma unroll
                for (int k = 0; k < kStages; ++k)
                    if (k == (int)fs) {
                        st_pos[k] = p.pos;
                        st_n[k] = p.n;
                    }
                ++issued;
            }
        }
    }
    bulk_wait_all<0>();
}

// ------------------------------------------------------------------------------------------------
// LSU kernel
// ------------------------------------------------------------------------------------------------
constexpr int kLsuThreads = 256;
constexpr int kLsuUnroll = 4;

// 16 B destination vectors, 16 B aligned source: straight streaming copy
__device__ __forceinline__ void contig_body_aligned(const char* __restrict__ s, char* __restrict__ d, uint64_t nvec) {
    const uint64_t i = threadIdx.x;
    const uint64_t step = (uint64_t)kLsuThreads * kLsuUnroll;
    for (uint64_t base = 0; base < nvec; base += step) {
        uint4 v[kLsuUnroll];
#pragma unroll
        for (int k = 0; k < kLsuUnroll; ++k) {
            const uint64_t j = base + i + (uint64_t)k * kLsuThreads;
            if (j < nvec) v[k] = ld_stream16(s + j * 16);
        }
#pragma unroll
        for (int k = 0; k < kLsuUnroll; ++k) {
            const uint64_t j = base + i + (uint64_t)k * kLsuThreads;
            if (j < nvec) st_stream16(d + j * 16, v[k]);
        }
    }
}

__device__ __forceinline__ uint4 ld_cached16(const void* p) {
    uint4 v;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}

// bytes [sh, sh+16) of the 32-byte concatenation lo:hi  (sh = 4*W + r, r in 0..3)
template <int W>
__device__ __forceinline__ uint4 shift_window(const uint4& lo, const uint4& hi, uint32_t rbits) {
    const uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    uint4 o;
    o.x = __funnelshift_r(w[W + 0], w[W + 1], rbits);
    o.y = __funnelshift_r(w[W + 1], w[W + 2], rbits);
    o.z = __funnelshift_r(w[W + 2], w[W + 3], rbits);
    o.w = __funnelshift_r(w[W + 3], w[(W + 4) & 7], rbits);
    return o;
}

// Source and destination disagree on their position inside a 16 B line (slab members are unpadded, so
// one odd-sized tensor shifts everything after it).  All global accesses stay 16 B wide and aligned: each
// output vector is cut out of two neighbouring aligned source vectors with funnel shifts.  The second
// load of every pair is the first load of the next thread, so it is served by L1.  The aligned loads may
// touch up to 15 bytes before/after the run, but never leave the 16 B lines that hold its bytes.
template <int W>
__device__ __forceinline__ void contig_body_shift_w(const char* __restrict__ s, char* __restrict__ d, uint64_t nvec,
                                                    uint32_t sh) {
    const char* a = s - sh;  // 16 B aligned
    const uint32_t rbits = (sh & 3) * 8;
    const uint64_t i = threadIdx.x;
    constexpr int kUnroll = 2;
    const uint64_t step = (uint64_t)kLsuThreads * kUnroll;
    for (uint64_t base = 0; base < nvec; base += step) {
        uint4 lo[kUnroll], hi[kUnroll];
#pragma unroll
        for (int k = 0; k < kUnroll; ++k) {
            const uint64_t j = base + i + (uint64_t)k * kLsuThreads;
            if (j < nvec) {
                lo[k] = ld_cached16(a + j * 16);
                hi[k] = ld_cached16(a + j * 16 + 16);
            }
        }
#pragma unroll
        for (int k = 0; k < kUnroll; ++k) {
            const uint64_t j = base + i + (uint64_t)k * kLsuThreads;
            if (j < nvec) st_stream16(d + j * 16, shift_window<W>(lo[k], hi[k], rbits));
        }
    }
}

__device__ __noinline__ void contig_body_shift(const char* s, char* d, uint64_t nvec) {
    const uint32_t sh = (uint32_t)(reinterpret_cast<uint64_t>(s) & 15);
    switch (sh >> 2) {
        case 0: contig_body_shift_w<0>(s, d, nvec, sh); break;
        case 1: contig_body_shift_w<1>(s, d, nvec, sh); break;
        case 2: contig_body_shift_w<2>(s, d, nvec, sh); break;
        default: contig_body_shift_w<3>(s, d, nvec, sh); break;
    }
}

__device__ __forceinline__ void tile_contig(const Member& m, uint32_t index) {
    uint64_t lo, hi;
    tile_range_contig(m, index, &lo, &hi);
    const char* s = reinterpret_cast<const char*>(m.src) + lo;
    char* d = reinterpret_cast<char*>(m.dst) + lo;
    const uint64_t n = hi - lo;
    uint64_t head = (16 - (reinterpret_cast<uint64_t>(d) & 15)) & 15;
    if (head > n) head = n;
    const uint64_t nvec = (n - head) >> 4;
    const uint64_t tail = n - head - (nvec << 4);
    // ragged edges: single bytes, warp 0 the head, warp 1 the tail
    if (threadIdx.x < head) d[threadIdx.x] = s[threadIdx.x];
    if (threadIdx.x >= 32 && threadIdx.x - 32 < tail) {
        const uint64_t o = head + (nvec << 4) + (threadIdx.x - 32);
        d[o] = s[o];
    }
    s += head;
    d += head;
    if ((reinterpret_cast<uint64_t>(s) & 15) == 0) contig_body_aligned(s, d, nvec);
    else contig_body_shift(s, d, nvec);
}

// row index -> byte offsets on both sides; the single-outer-dim case (2-D narrow / column shard) needs no division
__device__ __forceinline__ void row_offsets(const Member& m, uint64_t row, int64_t* so, int64_t* dofs) {
    if (m.nouter == 1) {
        *so = (int64_t)row * m.sstride[0];
        *dofs = (int64_t)row * m.dstride[0];
    } else {
        outer_offsets(m, row, so, dofs);
    }
}

// One granule (sizeof(T) bytes) per thread and step; kU independent loads are issued before the stores so that
// several requests per thread are in flight.  (row, col) of a thread's granule is divided out once per tile and
// then advanced incrementally: consecutive granules of a thread are a constant number of bytes apart.
template <typename T>
__device__ __forceinline__ void tile_strided_t(const Member& m, uint64_t lo, uint64_t hi) {
    constexpr int kU = sizeof(T) >= 8 ? 4 : 8;  // bytes in flight per SM = 3 CTAs x 256 thr x kU x sizeof(T)
    const char* sb = reinterpret_cast<const char*>(m.src);
    char* db = reinterpret_cast<char*>(m.dst);
    const uint64_t inner = m.inner;
    const uint64_t stride = (uint64_t)kLsuThreads * sizeof(T);
    uint64_t pos = lo + (uint64_t)threadIdx.x * sizeof(T);
    if (pos >= hi) return;
    uint64_t row, col, drow, dcol;
    if ((m.bytes >> 32) == 0) {
        const uint32_t in = (uint32_t)inner;
        row = (uint32_t)pos / in;
        col = (uint32_t)pos - (uint32_t)row * in;
        drow = (uint32_t)stride / in;
        dcol = (uint32_t)stride - (uint32_t)drow * in;
    } else {
        row = pos / inner;
        col = pos - row * inner;
        drow = stride / inner;
        dcol = stride - drow * inner;
    }
    while (pos < hi) {
        T v[kU];
        int64_t dst_off[kU];
#pragma unroll
        for (int k = 0; k < kU; ++k) {
            dst_off[k] = -1;
            if (pos < hi) {
                int64_t so, dofs;
                row_offsets(m, row, &so, &dofs);
                v[k] = __ldg(reinterpret_cast<const T*>(sb + so + (int64_t)col));
                dst_off[k] = dofs + (int64_t)col;
            }
            pos += stride;
            row += drow;
            col += dcol;
            if (col >= inner) {
                col -= inner;
                ++row;
            }
        }
#pragma unroll
        for (int k = 0; k < kU; ++k)
            if (dst_off[k] >= 0) *reinterpret_cast<T*>(db + dst_off[k]) = v[k];
    }
}

__device__ __noinline__ void tile_strided(const Member& m, uint32_t index) {
    uint64_t lo, hi;
    tile_range_lsu(m, index, &lo, &hi);
    switch (m.unit) {
        case 16: tile_strided_t<uint4>(m, lo, hi); break;
        case 8: tile_strided_t<uint2>(m, lo, hi); break;
        case 4: tile_strided_t<uint32_t>(m, lo, hi); break;
        case 2: tile_strided_t<uint16_t>(m, lo, hi); break;
        default: tile_strided_t<uint8_t>(m, lo, hi); break;
    }
}

// element i (compile-time constant after unrolling) of a 16 B vector, without taking the vector's address
template <typename T>
__device__ __forceinline__ T vec_get(const uint4& v, int i) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    if (sizeof(T) == 8) return (T)(((uint64_t)w[2 * i + 1] << 32) | w[2 * i]);
    if (sizeof(T) == 4) return (T)w[i];
    if (sizeof(T) == 2) return (T)((w[i >> 1] >> (16 * (i & 1))) & 0xffffu);
    return (T)((w[i >> 2] >> (8 * (i & 3))) & 0xffu);
}
template <typename T>
__device__ __forceinline__ void vec_put(uint32_t (&w)[4], int i, T x) {
    if (sizeof(T) == 8) {
        w[2 * i] = (uint32_t)((uint64_t)x);
        w[2 * i + 1] = (uint32_t)((uint64_t)x >> 32);
    } else if (sizeof(T) == 4) {
        w[i] = (uint32_t)x;
    } else if (sizeof(T) == 2) {
        w[i >> 1] |= (uint32_t)x << (16 * (i & 1));
    } else {
        w[i >> 2] |= (uint32_t)x << (8 * (i & 3));
    }
}

// ---- tiled transpose ---------------------------------------------------------------------------
// kModeTranspose: dim A is unit-stride on the source, dim B on the destination.  One tile = side x side elements of
// (A, B) for one index of the remaining dims: read with consecutive threads along A, write with consecutive threads
// along B, through a padded shared-memory tile — both sides see full-line accesses instead of an element gather.
template <typename T, int kA, int kB>
__device__ __forceinline__ void tile_transpose_t(const Member& m, uint32_t index, unsigned char* tbuf) {
    const uint32_t A = m.shift & 255, B = (m.shift >> 8) & 255;
    const uint64_t sA = (uint64_t)m.osize[A], sB = (uint64_t)m.osize[B];
    const uint32_t tilesA = (uint32_t)((sA + kA - 1) / kA), tilesB = (uint32_t)((sB + kB - 1) / kB);
    const uint32_t ib = index % tilesB;
    uint32_t rest = index / tilesB;
    const uint32_t ia = rest % tilesA;
    rest /= tilesA;
    int64_t so = 0, dofs = 0;
    for (int i = (int)m.nouter - 1; i >= 0; --i) {
        if ((uint32_t)i == A || (uint32_t)i == B) continue;
        const uint32_t sz = (uint32_t)m.osize[i];
        const uint32_t idx = rest % sz;
        rest /= sz;
        so += (int64_t)idx * m.sstride[i];
        dofs += (int64_t)idx * m.dstride[i];
    }
    const uint64_t a0 = (uint64_t)ia * kA, b0 = (uint64_t)ib * kB;
    const uint32_t na = (uint32_t)(sA - a0 < (uint64_t)kA ? sA - a0 : kA);
    const uint32_t nb = (uint32_t)(sB - b0 < (uint64_t)kB ? sB - b0 : kB);
    const int64_t ssB = m.sstride[B], dsA = m.dstride[A];
    const char* sp = reinterpret_cast<const char*>(m.src) + so + (int64_t)a0 * m.sstride[A] + (int64_t)b0 * ssB;
    char* dp = reinterpret_cast<char*>(m.dst) + dofs + (int64_t)a0 * dsA + (int64_t)b0 * m.dstride[B];
    T(*tile)[kA + 1] = reinterpret_cast<T(*)[kA + 1]>(tbuf);  // tile[b][a], one element of padding per row
    constexpr int V = 16 / (int)sizeof(T);  // elements per 16 B vector
    constexpr int kVecIn = kA / V;          // vectors per source row (along A)
    constexpr int kVecOut = kB / V;         // vectors per destination row (along B)
    constexpr int kIter = kB * kVecIn / kLsuThreads;
    static_assert(kB * kVecIn == kA * kVecOut && kIter * kLsuThreads == kB * kVecIn, "tile geometry");
    const bool full = na == (uint32_t)kA && nb == (uint32_t)kB && ((reinterpret_cast<uint64_t>(sp) | (uint64_t)ssB) & 15) == 0 &&
                      ((reinterpret_cast<uint64_t>(dp) | (uint64_t)dsA) & 15) == 0;
    if (full) {
        // interior tile: 16 B vectors on both global sides, all loads in flight before the first shared-memory store
        uint4 r[kIter];
#pragma unroll
        for (int k = 0; k < kIter; ++k) {
            const uint32_t idx = threadIdx.x + (uint32_t)k * kLsuThreads;
            r[k] = ld_stream16(sp + (int64_t)(idx / kVecIn) * ssB + (idx % kVecIn) * 16);
        }
#pragma unroll
        for (int k = 0; k < kIter; ++k) {
            const uint32_t idx = threadIdx.x + (uint32_t)k * kLsuThreads;
            const uint32_t b = idx / kVecIn, v = idx % kVecIn;
#pragma unroll
            for (int i = 0; i < V; ++i) tile[b][v * V + i] = vec_get<T>(r[k], i);
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < kIter; ++k) {
            const uint32_t idx = threadIdx.x + (uint32_t)k * kLsuThreads;
            const uint32_t a = idx / kVecOut, v = idx % kVecOut;
            uint32_t w[4] = {0, 0, 0, 0};
#pragma unroll
            for (int i = 0; i < V; ++i) vec_put<T>(w, i, tile[v * V + i][a]);
            st_stream16(dp + (int64_t)a * dsA + v * 16, make_uint4(w[0], w[1], w[2], w[3]));
        }
        return;  // the caller's loop synchronises before the tile buffer is reused
    }
    // edge tiles / unaligned bases: element accesses, still coalesced on both sides
    for (uint32_t e = threadIdx.x; e < nb * (uint32_t)kA; e += kLsuThreads) {
        const uint32_t b = e / kA, a = e % kA;
        if (a < na) tile[b][a] = __ldg(reinterpret_cast<const T*>(sp + (int64_t)b * ssB) + a);
    }
    __syncthreads();
    for (uint32_t e = threadIdx.x; e < na * (uint32_t)kB; e += kLsuThreads) {
        const uint32_t a = e / kB, b = e % kB;
        if (b < nb) reinterpret_cast<T*>(dp + (int64_t)a * dsA)[b] = tile[b][a];
    }
}

__device__ __noinline__ void tile_transpose(const Member& m, uint32_t index, unsigned char* tbuf) {
    switch (m.unit) {  // geometry = plan.h transpose_side_a / transpose_side_b
        case 8: tile_transpose_t<uint64_t, 64, 32>(m, index, tbuf); break;
        case 4: tile_transpose_t<uint32_t, 64, 64>(m, index, tbuf); break;
        case 2: tile_transpose_t<uint16_t, 128, 64>(m, index, tbuf); break;
        default: tile_transpose_t<uint8_t, 128, 128>(m, index, tbuf); break;
    }
}

// ---- fused cast -------------------------------------------------------------------------------
// dense, 16 B aligned, 2-byte <-> 4-byte float conversions: 8 elements per thread, 16 B accesses
template <bool kNarrow, bool kBf16>
__device__ __forceinline__ void cast_dense_vec(const char* __restrict__ s, char* __restrict__ d, uint64_t nelem) {
    const uint64_t ngroups = nelem >> 3;
    for (uint64_t g = threadIdx.x; g < ngroups; g += kLsuThreads) {
        if (kNarrow) {  // fp32 -> bf16 / fp16
            const uint4 a = ld_stream16(s + g * 32);
            const uint4 b = ld_stream16(s + g * 32 + 16);
            const float f[8] = {__uint_as_float(a.x), __uint_as_float(a.y), __uint_as_float(a.z), __uint_as_float(a.w),
                                __uint_as_float(b.x), __uint_as_float(b.y), __uint_as_float(b.z), __uint_as_float(b.w)};
            uint32_t o[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (kBf16) {
                    const __nv_bfloat162 p = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
                    o[i] = *reinterpret_cast<const uint32_t*>(&p);
                } else {
                    const __half2 p = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
                    o[i] = *reinterpret_cast<const uint32_t*>(&p);
                }
            }
            st_stream16(d + g * 16, make_uint4(o[0], o[1], o[2], o[3]));
        } else {  // bf16 / fp16 -> fp32
            const uint4 a = ld_stream16(s + g * 16);
            const uint32_t w[4] = {a.x, a.y, a.z, a.w};
            float f[8];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (kBf16) {
                    const float2 p = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]));
                    f[2 * i] = p.x;
                    f[2 * i + 1] = p.y;
                } else {
                    const float2 p = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
                    f[2 * i] = p.x;
                    f[2 * i + 1] = p.y;
                }
            }
            st_stream16(d + g * 32, make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3])));
            st_stream16(d + g * 32 + 16, make_uint4(__float_as_uint(f[4]), __float_as_uint(f[5]), __float_as_uint(f[6]), __float_as_uint(f[7])));
        }
    }
}

// dense, 16 B aligned {fp32, bf16, fp16} <-> float8: 16 elements per thread, one 16 B access on the float8 side and
// 16 B accesses on the wide side
template <uint32_t kWide>
__device__ __forceinline__ void ld16_as_f32(const char* s, float (&x)[16]) {
    if (kWide == TSNAP_F32) {
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const uint4 a = ld_stream16(s + 16 * v);
            x[4 * v] = __uint_as_float(a.x);
            x[4 * v + 1] = __uint_as_float(a.y);
            x[4 * v + 2] = __uint_as_float(a.z);
            x[4 * v + 3] = __uint_as_float(a.w);
        }
    } else {
#pragma unroll
        for (int v = 0; v < 2; ++v) {
            const uint4 a = ld_stream16(s + 16 * v);
            const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float2 f = kWide == TSNAP_BF16 ? __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]))
                                                     : __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
                x[8 * v + 2 * i] = f.x;
                x[8 * v + 2 * i + 1] = f.y;
            }
        }
    }
}
template <uint32_t kWide>
__device__ __forceinline__ void st16_from_f32(char* d, const float (&x)[16]) {
    if (kWide == TSNAP_F32) {
#pragma unroll
        for (int v = 0; v < 4; ++v)
            st_stream16(d + 16 * v, make_uint4(__float_as_uint(x[4 * v]), __float_as_uint(x[4 * v + 1]), __float_as_uint(x[4 * v + 2]),
                                               __float_as_uint(x[4 * v + 3])));
    } else {
#pragma unroll
        for (int v = 0; v < 2; ++v) {
            uint32_t o[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (kWide == TSNAP_BF16) {
                    const __nv_bfloat162 p = __floats2bfloat162_rn(x[8 * v + 2 * i], x[8 * v + 2 * i + 1]);
                    o[i] = *reinterpret_cast<const uint32_t*>(&p);
                } else {
                    const __half2 p = __floats2half2_rn(x[8 * v + 2 * i], x[8 * v + 2 * i + 1]);
                    o[i] = *reinterpret_cast<const uint32_t*>(&p);
                }
            }
            st_stream16(d + 16 * v, make_uint4(o[0], o[1], o[2], o[3]));
        }
    }
}
template <bool kNarrow, uint32_t kWide, uint32_t kFp8>
__device__ __forceinline__ void cast_fp8_vec(const char* __restrict__ s, char* __restrict__ d, uint64_t nelem) {
    constexpr uint32_t kWideSize = kWide == TSNAP_F32 ? 4 : 2;
    const uint64_t ngroups = nelem >> 4;
    for (uint64_t g = threadIdx.x; g < ngroups; g += kLsuThreads) {
        float x[16];
        uint32_t o[4];
        if (kNarrow) {
            ld16_as_f32<kWide>(s + g * 16 * kWideSize, x);
#pragma unroll
            for (int i = 0; i < 4; ++i)
                o[i] = (uint32_t)fp8_from_f32(x[4 * i], kFp8) | ((uint32_t)fp8_from_f32(x[4 * i + 1], kFp8) << 8) |
                       ((uint32_t)fp8_from_f32(x[4 * i + 2], kFp8) << 16) | ((uint32_t)fp8_from_f32(x[4 * i + 3], kFp8) << 24);
            st_stream16(d + g * 16, make_uint4(o[0], o[1], o[2], o[3]));
        } else {
            const uint4 a = ld_stream16(s + g * 16);
            o[0] = a.x, o[1] = a.y, o[2] = a.z, o[3] = a.w;
#pragma unroll
            for (int i = 0; i < 16; ++i) x[i] = fp8_to_f32((uint8_t)(o[i >> 2] >> (8 * (i & 3))), kFp8);
            st16_from_f32<kWide>(d + g * 16 * kWideSize, x);
        }
    }
}
template <bool kNarrow, uint32_t kWide>
__device__ __forceinline__ void cast_fp8_vec_of(uint32_t fp8, const char* s, char* d, uint64_t nelem) {
    if (fp8 == TSNAP_F8E4M3FN) cast_fp8_vec<kNarrow, kWide, TSNAP_F8E4M3FN>(s, d, nelem);
    else cast_fp8_vec<kNarrow, kWide, TSNAP_F8E5M2>(s, d, nelem);
}
// the float8 vector path for (src, dst), if it has one: the number of elements it converted (a multiple of 16)
__device__ __forceinline__ uint64_t cast_fp8_dense(uint32_t sdt, uint32_t ddt, const char* s, char* d, uint64_t nelem) {
    const bool narrow = is_fp8_dtype(ddt);
    const uint32_t wide = narrow ? sdt : ddt, fp8 = narrow ? ddt : sdt;
    if (!is_fp8_dtype(fp8) || !(wide == TSNAP_F32 || wide == TSNAP_BF16 || wide == TSNAP_F16)) return 0;
    if (narrow) {
        if (wide == TSNAP_F32) cast_fp8_vec_of<true, TSNAP_F32>(fp8, s, d, nelem);
        else if (wide == TSNAP_BF16) cast_fp8_vec_of<true, TSNAP_BF16>(fp8, s, d, nelem);
        else cast_fp8_vec_of<true, TSNAP_F16>(fp8, s, d, nelem);
    } else {
        if (wide == TSNAP_F32) cast_fp8_vec_of<false, TSNAP_F32>(fp8, s, d, nelem);
        else if (wide == TSNAP_BF16) cast_fp8_vec_of<false, TSNAP_BF16>(fp8, s, d, nelem);
        else cast_fp8_vec_of<false, TSNAP_F16>(fp8, s, d, nelem);
    }
    return nelem & ~uint64_t(15);
}

__device__ __noinline__ void tile_cast(const Member& m, uint32_t index) {
    uint64_t lo, hi;
    tile_range_lsu(m, index, &lo, &hi);
    uint64_t e0 = lo / m.dst_esz;
    const uint64_t e1 = hi / m.dst_esz;
    const char* sb = reinterpret_cast<const char*>(m.src);
    char* db = reinterpret_cast<char*>(m.dst);
    // fast path: one dense run on both sides, 16 B aligned, fp32 <-> {bf16, fp16} or {fp32, bf16, fp16} <-> float8
    if (m.nouter == 0 && ((m.src | m.dst) & 15) == 0) {
        const bool narrow = m.src_dtype == TSNAP_F32 && (m.dst_dtype == TSNAP_BF16 || m.dst_dtype == TSNAP_F16);
        const bool widen = m.dst_dtype == TSNAP_F32 && (m.src_dtype == TSNAP_BF16 || m.src_dtype == TSNAP_F16);
        if (narrow || widen) {
            const uint64_t n = e1 - e0;
            const char* s = sb + e0 * m.src_esz;
            char* d = db + e0 * m.dst_esz;
            if (narrow) {
                if (m.dst_dtype == TSNAP_BF16) cast_dense_vec<true, true>(s, d, n);
                else cast_dense_vec<true, false>(s, d, n);
            } else {
                if (m.src_dtype == TSNAP_BF16) cast_dense_vec<false, true>(s, d, n);
                else cast_dense_vec<false, false>(s, d, n);
            }
            e0 += n & ~uint64_t(7);  // the ragged tail (< 8 elements) goes through the scalar loop below
        } else {
            // {fp32, bf16, fp16} <-> float8; the ragged tail (< 16 elements) goes through the scalar loop below
            e0 += cast_fp8_dense(m.src_dtype, m.dst_dtype, sb + e0 * m.src_esz, db + e0 * m.dst_esz, e1 - e0);
        }
    }
    if (m.dst_dtype == TSNAP_QINT8 || m.dst_dtype == TSNAP_QUINT8) {
        // quantise-on-save: 1-byte destination elements, consecutive threads write consecutive bytes
        const bool is_signed = m.dst_dtype == TSNAP_QINT8;
        for (uint64_t e = e0 + threadIdx.x; e < e1; e += kLsuThreads) {
            const uint64_t row = e / m.inner, col = e - row * m.inner;
            int64_t so, dofs;
            outer_offsets(m, row, &so, &dofs);
            const float x = load_f32(sb + so + col * m.src_esz, m.src_dtype, true);
            reinterpret_cast<uint8_t*>(db + dofs)[col] = quantize_elem(x, m.q_scale, m.q_zero_point, is_signed);
        }
        if ((m.shift & 1) && hi == m.bytes && threadIdx.x < 16) {
            // the per-tensor trailer of T:serialization.py:278-310, byte by byte (the payload length is arbitrary)
            const unsigned char* t = threadIdx.x < 8 ? reinterpret_cast<const unsigned char*>(&m.q_scale) : reinterpret_cast<const unsigned char*>(&m.q_zero_point);
            db[m.bytes + threadIdx.x] = (char)t[threadIdx.x & 7];
        }
        return;
    }
    bool aligned = (m.dst % m.dst_esz) == 0, src_aligned = (m.src % m.src_esz) == 0;
    for (uint32_t i = 0; i < m.nouter; ++i) {
        aligned = aligned && ((uint64_t)m.dstride[i] % m.dst_esz) == 0;
        src_aligned = src_aligned && ((uint64_t)m.sstride[i] % m.src_esz) == 0;
    }
    for (uint64_t e = e0 + threadIdx.x; e < e1; e += kLsuThreads) {
        const uint64_t row = e / m.inner, col = e - row * m.inner;
        int64_t so, dofs;
        outer_offsets(m, row, &so, &dofs);
        convert_store(db + dofs + col * m.dst_esz, m.dst_dtype, sb + so + col * m.src_esz, m.src_dtype, src_aligned, aligned);
    }
}

// kMinBlocks = CTAs per SM the register allocation is bounded for: 3 caps it at 80 registers (the strided path then
// spills), 2 at 128, 6 at 40.  Three builds: strided tiles run on <2>, transpose tiles on <6> (a latency-bound
// load -> shared -> store cycle: more resident CTAs in different phases keep the memory system busy), every other mode
// on <3> (kernels.h; tools/kernel_cases.py times each mode).
template <int kMinBlocks>
__global__ void __launch_bounds__(kLsuThreads, kMinBlocks) tsnap_lsu_copy_kernel(const Member* __restrict__ members,
                                                                            const Tile* __restrict__ tiles, uint32_t ntiles) {
    __shared__ Member sm;
    __shared__ __align__(16) unsigned char tbuf[64 * 65 * 4 + 64];  // transpose tile: 64 x 65 x 4 B >= 64 x 129 x 2 B, 32 x 65 x 8 B, 128 x 129 B
    uint32_t loaded = 0xffffffffu;
    Tile next = blockIdx.x < ntiles ? tiles[blockIdx.x] : Tile{0, 0};
    for (uint32_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const Tile tl = next;
        if (t + gridDim.x < ntiles) next = tiles[t + gridDim.x];  // the descriptor of the next tile is in flight behind this tile's work
        // stage the member record in shared memory: every thread needs all of it (consecutive tiles of a CTA mostly
        // belong to the same member: reload only on change)
        __syncthreads();  // also fences the previous tile's use of sm / tbuf
        if (tl.member != loaded) {
            const uint32_t* g = reinterpret_cast<const uint32_t*>(members + tl.member);
            uint32_t* s = reinterpret_cast<uint32_t*>(&sm);
            for (uint32_t i = threadIdx.x; i < sizeof(Member) / 4; i += kLsuThreads) s[i] = g[i];
            loaded = tl.member;
            __syncthreads();
        }
        switch (sm.mode) {
            case kModeContig: tile_contig(sm, tl.index); break;
            case kModeStrided: tile_strided(sm, tl.index); break;
            case kModeCast: tile_cast(sm, tl.index); break;
            case kModeTranspose: tile_transpose(sm, tl.index, tbuf); break;
            default: {
                // unreachable: kernel_of sends every other mode to another kernel.  Kept for robustness: a
                // bulk-mode member, dense and 16B aligned on both sides
                uint64_t lo, hi;
                tile_range_lsu(sm, tl.index, &lo, &hi);
                contig_body_aligned(reinterpret_cast<const char*>(sm.src) + lo, reinterpret_cast<char*>(sm.dst) + lo,
                                    (hi - lo) >> 4);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// per-channel quantisation (kModeQChannel): statistics -> parameters -> quantising pack on save, dequantising
// scatter on restore.  A tile is a kTileLsu range of the member's destination bytes; a save tile is walked in chunks of
// 16 elements whose wire bytes are one 16 B-aligned vector (the body starts 8 B into a 256 B-aligned file image, so
// the first and last chunk of a tile may be shorter).
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kQChunk = 16;
constexpr uint32_t kQSmemChannels = 2048;  // members with at most this many channels aggregate a tile in shared memory

// (row, col) of the member's element walk and the byte offsets of the row on both sides
struct QWalk {
    uint64_t row, col;
    int64_t so, dofs;
};
__device__ __forceinline__ void qwalk_at(const Member& m, uint64_t e, QWalk& w) {
    w.row = e / m.inner;
    w.col = e - w.row * m.inner;
    outer_offsets(m, w.row, &w.so, &w.dofs);
}
__device__ __forceinline__ bool qwalk_next(const Member& m, QWalk& w) {  // true when a new row starts
    if (++w.col < m.inner) return false;
    w.col = 0;
    ++w.row;
    outer_offsets(m, w.row, &w.so, &w.dofs);
    return true;
}
// channel of the wire byte at `a`, and its position inside the channel's run of `inner` elements
__device__ __forceinline__ void qchan_at(const QChannel& q, uint64_t a, uint64_t* c, uint64_t* r) {
    const uint64_t off = a - q.body;
    if (((off | q.inner | q.channels) >> 32) == 0) {  // 32-bit division: every piece below 4 GiB
        const uint32_t t = (uint32_t)off / (uint32_t)q.inner;
        *r = (uint32_t)off - t * (uint32_t)q.inner;
        *c = t % (uint32_t)q.channels;
        return;
    }
    const uint64_t t = off / q.inner;
    *r = off - t * q.inner;
    *c = t % q.channels;
}
__device__ __forceinline__ void qchan_next(const QChannel& q, uint64_t* c, uint64_t* r) {
    if (++*r < q.inner) return;
    *r = 0;
    if (++*c == q.channels) *c = 0;
}
__device__ __forceinline__ uint64_t ld_u64_any(const char* p) {
    if ((reinterpret_cast<uintptr_t>(p) & 7) == 0) return *reinterpret_cast<const uint64_t*>(p);
    uint64_t v = 0;
    for (int i = 7; i >= 0; --i) v = (v << 8) | (uint8_t)p[i];
    return v;
}
__device__ __forceinline__ void st_u64_any(char* p, uint64_t v) {
    if ((reinterpret_cast<uintptr_t>(p) & 7) == 0) {
        *reinterpret_cast<uint64_t*>(p) = v;
        return;
    }
    for (int i = 0; i < 8; ++i) p[i] = (char)(v >> (8 * i));
}
__device__ __forceinline__ uint32_t ld_u32_any(const char* p) {
    if ((reinterpret_cast<uintptr_t>(p) & 3) == 0) return *reinterpret_cast<const uint32_t*>(p);
    uint32_t v = 0;
    for (int i = 3; i >= 0; --i) v = (v << 8) | (uint8_t)p[i];
    return v;
}
__device__ __forceinline__ void st_u32_any(char* p, uint32_t v) {
    if ((reinterpret_cast<uintptr_t>(p) & 3) == 0) {
        *reinterpret_cast<uint32_t*>(p) = v;
        return;
    }
    for (int i = 0; i < 4; ++i) p[i] = (char)(v >> (8 * i));
}

// The source elements of save chunk [e, e + n) as fp32 (the value the quantiser reads); 16 B loads when the chunk is
// a full, 16 B-aligned piece of one dense run.
__device__ __forceinline__ void qload_chunk(const Member& m, uint64_t e, uint32_t n, float (&x)[kQChunk]) {
    const char* sb = reinterpret_cast<const char*>(m.src);
    if (m.nouter == 0 && n == kQChunk && ((m.src + e * m.src_esz) & 15) == 0 && m.src_dtype != TSNAP_F64) {
        const uint4* p = reinterpret_cast<const uint4*>(sb + e * m.src_esz);
        if (m.src_dtype == TSNAP_F32) {
#pragma unroll
            for (int v = 0; v < 4; ++v) {
                const uint4 a = ld_stream16(p + v);
                x[4 * v] = __uint_as_float(a.x);
                x[4 * v + 1] = __uint_as_float(a.y);
                x[4 * v + 2] = __uint_as_float(a.z);
                x[4 * v + 3] = __uint_as_float(a.w);
            }
        } else {
#pragma unroll
            for (int v = 0; v < 2; ++v) {
                const uint4 a = ld_stream16(p + v);
                const uint32_t w[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const float2 f = m.src_dtype == TSNAP_BF16 ? __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]))
                                                               : __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
                    x[8 * v + 2 * i] = f.x;
                    x[8 * v + 2 * i + 1] = f.y;
                }
            }
        }
        return;
    }
    QWalk w;
    qwalk_at(m, e, w);
#pragma unroll
    for (uint32_t i = 0; i < kQChunk; ++i) {
        if (i < n) {
            x[i] = load_f32(sb + w.so + w.col * m.src_esz, m.src_dtype, true);
            qwalk_next(m, w);
        }
    }
}

// chunk k of a save tile [e0, e1): elements [*ce, *ce + *cn), cut at the 16 B boundaries of the wire bytes
__device__ __forceinline__ bool qsave_chunk(const Member& m, uint64_t e0, uint64_t e1, uint64_t k, uint64_t* ce, uint32_t* cn) {
    const uint64_t a0 = m.dst + e0, first = (a0 & ~uint64_t(15)) + 16 * k;
    const uint64_t lo = first > a0 ? first : a0;
    uint64_t hi = first + 16;
    if (hi > m.dst + e1) hi = m.dst + e1;
    if (lo >= hi) return false;
    *ce = lo - m.dst;
    *cn = (uint32_t)(hi - lo);
    return true;
}

// one run of equal channel: fold (kmin, kmax) into the shared table or the member's key slots.  Lanes holding the same
// channel are combined first (all 32 lanes call this together; a lane with nothing to add passes c = ~0).
__device__ __forceinline__ void qstats_flush(uint64_t c, int32_t kmin, int32_t kmax, int* smem, int* keys) {
    const unsigned peers = __match_any_sync(0xffffffffu, c);
    const int mn = __reduce_min_sync(peers, kmin), mx = __reduce_max_sync(peers, kmax);
    if (c != ~uint64_t(0) && (threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) {
        int* slot = smem ? smem + 2 * c : keys + 2 * c;
        if (mn < 0) atomicMin(slot, mn);
        if (mx > 0) atomicMax(slot + 1, mx);
    }
}

__global__ void __launch_bounds__(kLsuThreads) tsnap_qstats_kernel(const Member* __restrict__ members, const QChannel* __restrict__ qch,
                                                                   const Tile* __restrict__ tiles, uint32_t ntiles) {
    __shared__ int table[2 * kQSmemChannels];
    __shared__ int pacc[2 * kQChunk * kLsuThreads];  // per thread: (min, max) of its 16 chunk positions, see `periodic`
    for (uint32_t i = threadIdx.x; i < 2 * kQSmemChannels; i += kLsuThreads) table[i] = 0;
    int* const pmin = pacc + threadIdx.x;                        // position i at pmin[i * kLsuThreads]
    int* const pmax = pacc + kQChunk * kLsuThreads + threadIdx.x;
    for (uint32_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const Tile tl = tiles[t];
        const Member& m = members[tl.member];
        const QChannel q = qch[m.q_zero_point];
        uint64_t lo, hi;
        tile_range_lsu(m, tl.index, &lo, &hi);
        const bool shared = q.channels <= kQSmemChannels;
        int* keys = reinterpret_cast<int*>(q.keys);
        __syncthreads();  // the table is clean
        // every lane runs the same number of iterations so that qstats_flush is called by whole warps
        const uint64_t nchunks = (((m.dst + hi + 15) & ~uint64_t(15)) - ((m.dst + lo) & ~uint64_t(15))) / 16;
        const uint64_t iters = (nchunks + kLsuThreads - 1) / kLsuThreads;
        // When channels x inner divides the stride between a thread's chunks (16 x kLsuThreads wire bytes), every full
        // chunk of the thread covers the same 16 channel positions: they are accumulated in the thread's own shared-memory
        // slots, without atomics (axis -1 of a [N, 1024] weight would otherwise cost two atomics per element).  Shared
        // rather than registers: 32 more registers would cost a resident CTA per SM on every member.
        const bool periodic = (kQChunk * kLsuThreads) % (q.channels * q.inner) == 0;
        uint64_t pbase = ~uint64_t(0);  // wire address of this thread's full chunks, modulo the period
#pragma unroll
        for (uint32_t i = 0; i < kQChunk; ++i) pmin[i * kLsuThreads] = pmax[i * kLsuThreads] = 0;
        for (uint64_t it = 0; it < iters; ++it) {
            uint64_t ce = 0, c = ~uint64_t(0), r = 0;
            uint32_t cn = 0;
            int32_t kmin = 0, kmax = 0;
            if (qsave_chunk(m, lo, hi, it * kLsuThreads + threadIdx.x, &ce, &cn)) {
                float x[kQChunk];
                qload_chunk(m, ce, cn, x);
                if (periodic && cn == kQChunk && ((m.dst + ce) & 15) == 0) {
                    pbase = m.dst + ce;
#pragma unroll
                    for (uint32_t i = 0; i < kQChunk; ++i) {
                        const int32_t k = qkey(x[i]);
                        pmin[i * kLsuThreads] = min(pmin[i * kLsuThreads], k);
                        pmax[i * kLsuThreads] = max(pmax[i * kLsuThreads], k);
                    }
                    cn = 0;  // nothing left for the run-by-run path below
                }
                if (cn) qchan_at(q, m.dst + ce, &c, &r);
#pragma unroll
                for (uint32_t i = 0; i < kQChunk; ++i) {
                    if (i < cn) {
                        const int32_t k = qkey(x[i]);
                        kmin = min(kmin, k);
                        kmax = max(kmax, k);
                        if (i + 1 < cn && r + 1 == q.inner) {  // the next element starts another channel: this run is complete
                            int* slot = shared ? table + 2 * c : keys + 2 * c;
                            if (kmin < 0) atomicMin(slot, kmin);
                            if (kmax > 0) atomicMax(slot + 1, kmax);
                            kmin = kmax = 0;
                        }
                        qchan_next(q, &c, &r);
                    }
                }
                // qchan_next moved past the last element: step back to the channel of the pending run
                if (cn) c = (r == 0 ? (c == 0 ? q.channels - 1 : c - 1) : c);
            }
            if (__any_sync(0xffffffffu, c != ~uint64_t(0))) qstats_flush(c, kmin, kmax, shared ? table : nullptr, keys);
        }
        if (pbase != ~uint64_t(0)) {
            uint64_t c, r;
            qchan_at(q, pbase, &c, &r);
            for (uint32_t i = 0; i < kQChunk; ++i) {
                int* slot = shared ? table + 2 * c : keys + 2 * c;
                if (pmin[i * kLsuThreads] < 0) atomicMin(slot, pmin[i * kLsuThreads]);
                if (pmax[i * kLsuThreads] > 0) atomicMax(slot + 1, pmax[i * kLsuThreads]);
                qchan_next(q, &c, &r);
            }
        }
        if (shared) {
            __syncthreads();
            // channels the tile touched: one contiguous range of the wire modulo C
            const uint64_t c_lo = (m.dst + lo - q.body) / q.inner, c_hi = (m.dst + hi - 1 - q.body) / q.inner;
            const uint64_t span = c_hi - c_lo + 1 < q.channels ? c_hi - c_lo + 1 : q.channels;
            for (uint64_t j = threadIdx.x; j < span; j += kLsuThreads) {
                const uint64_t c = (c_lo + j) % q.channels;
                const int mn = table[2 * c], mx = table[2 * c + 1];
                if (mn < 0) atomicMin(keys + 2 * c, mn);
                if (mx > 0) atomicMax(keys + 2 * c + 1, mx);
                table[2 * c] = table[2 * c + 1] = 0;
            }
        }
    }
}

// finalises each channel's keys into (scale: f64, zero_point: i64) in place, copies them into the wire image and writes
// the axis header; a NaN / Inf channel raises *nonfinite.  kFp8 (kModeQChannelFp8): the f32 scale of fp8_scale_of
// instead, in the key slot and in the wire image.
template <bool kFp8>
__global__ void __launch_bounds__(kLsuThreads) tsnap_qparams_kernel(const Member* __restrict__ members, const QChannel* __restrict__ qch,
                                                                    const Tile* __restrict__ tiles, uint32_t ntiles, int* nonfinite) {
    for (uint32_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const Tile tl = tiles[t];
        const Member& m = members[tl.member];
        const QChannel q = qch[m.q_zero_point];
        const bool is_signed = m.dst_dtype == TSNAP_QINT8;
        const uint64_t c0 = (uint64_t)tl.index * kQChannelsPerTile;
        const uint64_t c1 = c0 + kQChannelsPerTile < q.channels ? c0 + kQChannelsPerTile : q.channels;
        char* params = reinterpret_cast<char*>(q.params);
        if constexpr (kFp8) {
            for (uint64_t c = c0 + threadIdx.x; c < c1; c += kLsuThreads) {
                int* k = reinterpret_cast<int*>(q.keys) + 2 * c;
                float s;
                if (!fp8_scale_of(k[0], k[1], m.dst_dtype, &s)) {
                    *nonfinite = 1;
                    s = __int_as_float(0x7fc00000);
                }
                k[0] = __float_as_int(s);  // the pack divides by it
                st_u32_any(params + 4 * c, __float_as_uint(s));
            }
        } else for (uint64_t c = c0 + threadIdx.x; c < c1; c += kLsuThreads) {
            int* k = reinterpret_cast<int*>(q.keys) + 2 * c;
            double scale;
            int64_t zp;
            if (!qparams_of(k[0], k[1], is_signed, &scale, &zp)) {
                *nonfinite = 1;
                scale = __longlong_as_double(0x7ff8000000000000ll);
                zp = 0;
            }
            // the quantising pack reads (1 / scale: f32, zero_point: i32) per element: 8 B per channel, scales behind them
            k[0] = __float_as_int((float)(1.0 / scale));
            k[1] = (int)zp;
            reinterpret_cast<double*>(q.keys + 8 * q.channels)[c] = scale;
            st_u64_any(params + 8 * c, (uint64_t)__double_as_longlong(scale));
            st_u64_any(params + 8 * (q.channels + c), (uint64_t)zp);
        }
        if (tl.index == 0 && threadIdx.x == 0) st_u64_any(reinterpret_cast<char*>(q.body) - 8, (uint64_t)q.axis);
    }
}

// One kModeQChannelFp8 tile, [lo, hi) of the member's destination bytes; kDt is the float8 wire dtype.
// Save: float8(clamp(x / s, -FMAX, FMAX)) with fp8_quantize's IEEE division, 16 elements and one 16 B store per thread
// as in the int8 pack.  Restore: fp32(q) * s, converted once to the destination dtype.
template <uint32_t kDt>
__device__ __forceinline__ void qchannel_fp8_tile(const Member& m, const QChannel& q, uint64_t lo, uint64_t hi) {
    if (q.save) {
        const float* sk = reinterpret_cast<const float*>(q.keys);  // (s, unused) per channel, from tsnap_qparams_kernel<true>
        char* db = reinterpret_cast<char*>(m.dst);
        uint64_t ce;
        uint32_t cn;
        for (uint64_t k = threadIdx.x; qsave_chunk(m, lo, hi, k, &ce, &cn); k += kLsuThreads) {
            float x[kQChunk];
            qload_chunk(m, ce, cn, x);
            uint64_t c, r;
            qchan_at(q, m.dst + ce, &c, &r);
            uint64_t loaded = ~uint64_t(0);
            float s = 1.0f;
            uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
            for (uint32_t i = 0; i < kQChunk; ++i) {
                if (i < cn) {
                    if (c != loaded) {
                        s = sk[2 * c];
                        loaded = c;
                    }
                    o[i >> 2] |= (uint32_t)fp8_quantize(x[i], s, kDt) << (8 * (i & 3));
                    qchan_next(q, &c, &r);
                }
            }
            if (cn == kQChunk) {
                st_stream16(db + ce, make_uint4(o[0], o[1], o[2], o[3]));
            } else {
                for (uint32_t i = 0; i < cn; ++i) db[ce + i] = (char)(o[i >> 2] >> (8 * (i & 3)));
            }
        }
        return;
    }
    const char* sb = reinterpret_cast<const char*>(m.src);
    char* db = reinterpret_cast<char*>(m.dst);
    const char* params = reinterpret_cast<const char*>(q.params);  // f32 scales at any alignment
    bool aligned = (m.dst % m.dst_esz) == 0;
    for (uint32_t i = 0; i < m.nouter; ++i) aligned = aligned && ((uint64_t)m.dstride[i] % m.dst_esz) == 0;
    const uint64_t e0 = lo / m.dst_esz, e1 = hi / m.dst_esz;
    if (m.nouter == 0 && m.dst_dtype != TSNAP_F64 && ((m.dst + e0 * m.dst_esz) & 15) == 0 && ((m.src + e0) & 3) == 0) {
        // one dense run on both sides: 4 elements per thread and step, a 4-byte load and one 8 or 16-byte store
        const uint64_t ngroups = (e1 - e0) / 4;
        uint64_t loaded = ~uint64_t(0);
        float s = 1.0f;
        for (uint64_t g = threadIdx.x; g < ngroups; g += kLsuThreads) {
            const uint64_t e = e0 + 4 * g;
            const uint32_t w = *reinterpret_cast<const uint32_t*>(sb + e);
            uint64_t c, r;
            qchan_at(q, m.src + e, &c, &r);
            float f[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (c != loaded) {
                    s = __uint_as_float(ld_u32_any(params + 4 * c));
                    loaded = c;
                }
                f[i] = fp8_dequantize((uint8_t)(w >> (8 * i)), kDt, s);
                qchan_next(q, &c, &r);
            }
            char* p = db + e * m.dst_esz;
            if (m.dst_dtype == TSNAP_F32) {
                *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
            } else {
                uint16_t h[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) h[i] = f16_or_bf16_from_f32(f[i], m.dst_dtype);
                *reinterpret_cast<uint2*>(p) = make_uint2(h[0] | ((uint32_t)h[1] << 16), h[2] | ((uint32_t)h[3] << 16));
            }
        }
        if (threadIdx.x == 0) {  // the ragged tail (< 4 elements)
            for (uint64_t e = e0 + 4 * ngroups; e < e1; ++e) {
                uint64_t c, r;
                qchan_at(q, m.src + e, &c, &r);
                const float f = fp8_dequantize((uint8_t)sb[e], kDt, __uint_as_float(ld_u32_any(params + 4 * c)));
                store_f32(db + e * m.dst_esz, m.dst_dtype, f, true);
            }
        }
        return;
    }
    for (uint64_t e = e0 + (uint64_t)threadIdx.x * kQChunk; e < e1; e += (uint64_t)kLsuThreads * kQChunk) {
        const uint32_t n = e1 - e < kQChunk ? (uint32_t)(e1 - e) : kQChunk;
        QWalk w;
        qwalk_at(m, e, w);
        uint64_t c, r;
        qchan_at(q, m.src + w.so + w.col, &c, &r);
        for (uint32_t i = 0; i < n; ++i) {
            const float s = __uint_as_float(ld_u32_any(params + 4 * c));
            store_f32(db + w.dofs + w.col * m.dst_esz, m.dst_dtype, fp8_dequantize((uint8_t)sb[w.so + w.col], kDt, s), aligned);
            if (qwalk_next(m, w)) qchan_at(q, m.src + w.so, &c, &r);
            else qchan_next(q, &c, &r);
        }
    }
}

// torch's per-channel quantiser on the device (ATen/native/quantized/cuda/AffineQuantizer.cu): the same rounding as
// quantize_elem, with the channel's parameters.  kFp8: the scaled float8 tiles of kModeQChannelFp8 instead.
template <bool kFp8>
__global__ void __launch_bounds__(kLsuThreads) tsnap_qchannel_kernel(const Member* __restrict__ members, const QChannel* __restrict__ qch,
                                                                     const Tile* __restrict__ tiles, uint32_t ntiles) {
    for (uint32_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const Tile tl = tiles[t];
        const Member& m = members[tl.member];
        const QChannel q = qch[m.q_zero_point];
        uint64_t lo, hi;
        tile_range_lsu(m, tl.index, &lo, &hi);
        if constexpr (kFp8) {
            if ((q.save ? m.dst_dtype : m.src_dtype) == TSNAP_F8E4M3FN) qchannel_fp8_tile<TSNAP_F8E4M3FN>(m, q, lo, hi);
            else qchannel_fp8_tile<TSNAP_F8E5M2>(m, q, lo, hi);
            continue;
        }
        if (q.save) {
            const bool is_signed = m.dst_dtype == TSNAP_QINT8;
            const uint2* kp = reinterpret_cast<const uint2*>(q.keys);                       // (1 / scale: f32, zero_point: i32)
            const double* scales = reinterpret_cast<const double*>(q.keys + 8 * q.channels);
            char* db = reinterpret_cast<char*>(m.dst);
            uint64_t ce;
            uint32_t cn;
            for (uint64_t k = threadIdx.x; qsave_chunk(m, lo, hi, k, &ce, &cn); k += kLsuThreads) {
                float x[kQChunk];
                qload_chunk(m, ce, cn, x);
                uint64_t c, r;
                qchan_at(q, m.dst + ce, &c, &r);
                uint64_t loaded = ~uint64_t(0);
                float inv = 1.0f;
                int zp = 0;
                uint32_t o[4] = {0, 0, 0, 0};
#pragma unroll
                for (uint32_t i = 0; i < kQChunk; ++i) {
                    if (i < cn) {
                        if (c != loaded) {
                            const uint2 p = kp[c];
                            inv = __uint_as_float(p.x);
                            zp = (int)p.y;
                            loaded = c;
                        }
                        // nearbyint(x / scale) without a division: x * fp32(1 / scale) is within 3e-5 of the quotient
                        // (|x / scale| <= 255 under the default rule), so its rounding is the quotient's unless it lies
                        // that close to a tie — then the division decides, as quantize_elem does it
                        const float y = x[i] * inv;
                        const float t = rintf(y);
                        int v = fabsf(fabsf(y - t) - 0.5f) > 1e-4f && isfinite(y) ? (int)t : (int)nearbyint((double)x[i] / scales[c]);
                        v += zp;
                        const int qlo = is_signed ? -128 : 0, qhi = is_signed ? 127 : 255;
                        v = v < qlo ? qlo : (v > qhi ? qhi : v);
                        o[i >> 2] |= (uint32_t)(uint8_t)(int8_t)v << (8 * (i & 3));
                        qchan_next(q, &c, &r);
                    }
                }
                if (cn == kQChunk) {
                    st_stream16(db + ce, make_uint4(o[0], o[1], o[2], o[3]));  // the wire side of a save is dense
                } else {
                    for (uint32_t i = 0; i < cn; ++i) db[ce + i] = (char)(o[i >> 2] >> (8 * (i & 3)));
                }
            }
            continue;
        }
        // restore: float((q - zero_point) * scale) in double, converted to the destination dtype
        const bool is_signed = m.src_dtype == TSNAP_QINT8;
        const char* sb = reinterpret_cast<const char*>(m.src);
        char* db = reinterpret_cast<char*>(m.dst);
        const char* params = reinterpret_cast<const char*>(q.params);
        bool aligned = (m.dst % m.dst_esz) == 0;
        for (uint32_t i = 0; i < m.nouter; ++i) aligned = aligned && ((uint64_t)m.dstride[i] % m.dst_esz) == 0;
        const uint64_t e0 = lo / m.dst_esz, e1 = hi / m.dst_esz;
        if (m.nouter == 0 && m.dst_dtype != TSNAP_F64 && ((m.dst + e0 * m.dst_esz) & 15) == 0 && ((m.src + e0) & 3) == 0) {
            // one dense run on both sides: 4 elements per thread and step, a 4-byte load and one 8 or 16-byte store
            const uint64_t ngroups = (e1 - e0) / 4;
            uint64_t loaded = ~uint64_t(0);
            double scale = 1.0, zp = 0.0;
            for (uint64_t g = threadIdx.x; g < ngroups; g += kLsuThreads) {
                const uint64_t e = e0 + 4 * g;
                const uint32_t w = *reinterpret_cast<const uint32_t*>(sb + e);
                uint64_t c, r;
                qchan_at(q, m.src + e, &c, &r);
                float f[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    if (c != loaded) {
                        scale = __longlong_as_double((long long)ld_u64_any(params + 8 * c));
                        zp = (double)(int64_t)ld_u64_any(params + 8 * (q.channels + c));
                        loaded = c;
                    }
                    const uint32_t raw = (w >> (8 * i)) & 255;
                    const double v = is_signed ? (double)(int8_t)raw : (double)raw;
                    f[i] = (float)((v - zp) * scale);
                    qchan_next(q, &c, &r);
                }
                char* p = db + e * m.dst_esz;
                if (m.dst_dtype == TSNAP_F32) {
                    *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
                } else {
                    uint16_t h[4];
#pragma unroll
                    for (int i = 0; i < 4; ++i) h[i] = f16_or_bf16_from_f32(f[i], m.dst_dtype);
                    *reinterpret_cast<uint2*>(p) = make_uint2(h[0] | ((uint32_t)h[1] << 16), h[2] | ((uint32_t)h[3] << 16));
                }
            }
            if (threadIdx.x == 0) {  // the ragged tail (< 4 elements)
                for (uint64_t e = e0 + 4 * ngroups; e < e1; ++e) {
                    uint64_t c, r;
                    qchan_at(q, m.src + e, &c, &r);
                    const float f = dequantize((uint8_t)sb[e], is_signed, (int64_t)ld_u64_any(params + 8 * (q.channels + c)),
                                               __longlong_as_double((long long)ld_u64_any(params + 8 * c)));
                    store_f32(db + e * m.dst_esz, m.dst_dtype, f, true);
                }
            }
            continue;
        }
        for (uint64_t e = e0 + (uint64_t)threadIdx.x * kQChunk; e < e1; e += (uint64_t)kLsuThreads * kQChunk) {
            const uint32_t n = e1 - e < kQChunk ? (uint32_t)(e1 - e) : kQChunk;
            QWalk w;
            qwalk_at(m, e, w);
            uint64_t c, r;
            qchan_at(q, m.src + w.so + w.col, &c, &r);
            for (uint32_t i = 0; i < n; ++i) {
                const double scale = __longlong_as_double((long long)ld_u64_any(params + 8 * c));
                const int64_t zp = (int64_t)ld_u64_any(params + 8 * (q.channels + c));
                store_f32(db + w.dofs + w.col * m.dst_esz, m.dst_dtype, dequantize((uint8_t)sb[w.so + w.col], is_signed, zp, scale), aligned);
                if (qwalk_next(m, w)) qchan_at(q, m.src + w.so, &c, &r);
                else qchan_next(q, &c, &r);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
// Ring geometry of the copy-engine kernels: two 48 KiB stages per one-warp CTA, two CTAs per SM (192 KiB of the
// H100's 228 KiB of shared memory per SM).  On an H100 SXM (700 W) it moves a dense 1 GiB member at 2.82-2.83 TB/s
// of algorithmic traffic (tools/kernel_cases.py, CUDA events), 0.84 of the 3.35 TB/s data-sheet HBM3 bandwidth; the
// first version's 3 x 16 KiB ring with 4 CTAs per SM measured the same.
constexpr int kRingStages = 2, kRingStageBytes = 49152, kRingCtasPerSm = 2;
constexpr int kBulkSmem = kRingStages * kRingStageBytes + kRingStages * 8;
constexpr int kRowsSmem = kRingStages * kRingStageBytes + kRingStages * (int)sizeof(Member) + kRingStages * 8;

// resident CTAs per SM of the three builds of the LSU kernel (kKernelLsu, kKernelLsuStrided, kKernelLsuTranspose), from
// the occupancy calculator: each persistent grid is exactly one wave
static int g_lsu_ctas_per_sm[3] = {3, 2, 6};
// kKernelQStats .. kKernelQChannelFp8 (from the occupancy calculator)
static int g_qchannel_ctas_per_sm[5] = {2, 2, 2, 2, 2};

cudaError_t init_kernels() {
    cudaError_t e = cudaFuncSetAttribute(tsnap_bulk_copy_kernel<kRingStages, kRingStageBytes>, cudaFuncAttributeMaxDynamicSharedMemorySize, kBulkSmem);
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(tsnap_rows_copy_kernel<kRingStages, kRingStageBytes>, cudaFuncAttributeMaxDynamicSharedMemorySize, kRowsSmem);
    if (e == cudaSuccess) {
        int n = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, tsnap_lsu_copy_kernel<3>, kLsuThreads, 0) == cudaSuccess && n > 0) g_lsu_ctas_per_sm[0] = n;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, tsnap_lsu_copy_kernel<2>, kLsuThreads, 0) == cudaSuccess && n > 0) g_lsu_ctas_per_sm[1] = n;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, tsnap_lsu_copy_kernel<6>, kLsuThreads, 0) == cudaSuccess && n > 0) g_lsu_ctas_per_sm[2] = n;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, tsnap_qstats_kernel, kLsuThreads, 0) == cudaSuccess && n > 0) g_qchannel_ctas_per_sm[0] = n;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, tsnap_qparams_kernel<false>, kLsuThreads, 0) == cudaSuccess && n > 0) g_qchannel_ctas_per_sm[1] = n;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, tsnap_qparams_kernel<true>, kLsuThreads, 0) == cudaSuccess && n > 0) g_qchannel_ctas_per_sm[2] = n;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, tsnap_qchannel_kernel<false>, kLsuThreads, 0) == cudaSuccess && n > 0) g_qchannel_ctas_per_sm[3] = n;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, tsnap_qchannel_kernel<true>, kLsuThreads, 0) == cudaSuccess && n > 0) g_qchannel_ctas_per_sm[4] = n;
    }
    return e;
}

cudaError_t launch_kernel(Kernel k, const Member* d_members, const Tile* d_tiles, const TmaPair* d_maps, uint32_t ntiles,
                          int sm_count, cudaStream_t stream) {
    if (ntiles == 0) return cudaSuccess;
    if (k == kKernelRowsTma || k == kKernelTransposeTma) return launch_tma_kernel(k, d_members, d_tiles, d_maps, ntiles, sm_count, stream);
    const bool ring = k == kKernelBulk || k == kKernelRows;
    uint32_t grid = (uint32_t)sm_count * (uint32_t)(ring ? kRingCtasPerSm : g_lsu_ctas_per_sm[k - kKernelLsu]);
    if (grid > ntiles) grid = ntiles;
    switch (k) {
        case kKernelBulk: tsnap_bulk_copy_kernel<kRingStages, kRingStageBytes><<<grid, 32, kBulkSmem, stream>>>(d_members, d_tiles, ntiles); break;
        case kKernelRows: tsnap_rows_copy_kernel<kRingStages, kRingStageBytes><<<grid, 32, kRowsSmem, stream>>>(d_members, d_tiles, ntiles); break;
        case kKernelLsuStrided: tsnap_lsu_copy_kernel<2><<<grid, kLsuThreads, 0, stream>>>(d_members, d_tiles, ntiles); break;
        case kKernelLsuTranspose: tsnap_lsu_copy_kernel<6><<<grid, kLsuThreads, 0, stream>>>(d_members, d_tiles, ntiles); break;
        default: tsnap_lsu_copy_kernel<3><<<grid, kLsuThreads, 0, stream>>>(d_members, d_tiles, ntiles); break;
    }
    return cudaGetLastError();
}

cudaError_t launch_qchannel_kernel(Kernel k, const Member* d_members, const QChannel* d_qch, const Tile* d_tiles, uint32_t ntiles,
                                   int* nonfinite, int sm_count, cudaStream_t stream) {
    if (ntiles == 0) return cudaSuccess;
    uint32_t grid = (uint32_t)sm_count * (uint32_t)g_qchannel_ctas_per_sm[k - kKernelQStats];
    if (grid > ntiles) grid = ntiles;
    switch (k) {
        case kKernelQStats: tsnap_qstats_kernel<<<grid, kLsuThreads, 0, stream>>>(d_members, d_qch, d_tiles, ntiles); break;
        case kKernelQParams: tsnap_qparams_kernel<false><<<grid, kLsuThreads, 0, stream>>>(d_members, d_qch, d_tiles, ntiles, nonfinite); break;
        case kKernelQParamsFp8: tsnap_qparams_kernel<true><<<grid, kLsuThreads, 0, stream>>>(d_members, d_qch, d_tiles, ntiles, nonfinite); break;
        case kKernelQChannelFp8: tsnap_qchannel_kernel<true><<<grid, kLsuThreads, 0, stream>>>(d_members, d_qch, d_tiles, ntiles); break;
        default: tsnap_qchannel_kernel<false><<<grid, kLsuThreads, 0, stream>>>(d_members, d_qch, d_tiles, ntiles); break;
    }
    return cudaGetLastError();
}

}  // namespace tsnap
