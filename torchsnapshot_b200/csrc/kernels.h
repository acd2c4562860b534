#pragma once
#include <cuda_runtime.h>

#include "plan.h"

namespace tsnap {
// The copy kernels, in the order a wave launches them; each runs one tile list of the wave.  Fractions of the H100 SXM
// data-sheet HBM3 bandwidth (3.35 TB/s) measured with tools/kernel_cases.py; the LSU kernel has three builds whose
// register bound sets the resident CTAs per SM.
enum Kernel {
    kKernelBulk,          // kModeBulk: copy-engine ring over dense runs (kernels.cu)
    kKernelRows,          // kModeRows: one copy-engine request per run (kernels.cu)
    kKernelRowsTma,       // kModeRowsTma: tensor-map boxes of many short runs (transpose_tma.cu)
    kKernelQStats,        // kModeQChannel saves: per-channel min / max of the source into the wave's key slots
    kKernelQParams,       // kModeQChannel saves: keys -> (scale, zero_point), the wire image's parameters and axis header
    kKernelQParamsFp8,    // kModeQChannelFp8 saves: keys -> f32 scale, the wire image's scales and axis header
    kKernelQChannel,      // kModeQChannel: quantising pack (16 B of int8 per thread) / dequantising scatter
    kKernelQChannelFp8,   // kModeQChannelFp8: scaled float8 pack (16 B of float8 per thread) / dequantising scatter
    kKernelLsu,           // kModeContig, kModeCast: 3 CTAs/SM, 80 registers: unaligned dense runs 0.76, fp32 -> bf16 casts 0.87
    kKernelLsuStrided,    // kModeStrided: 2 CTAs/SM, 128 registers: the strided gather keeps 8 independent 16 B loads per
                          // thread in flight without spilling (0.68 on 128 B runs)
    kKernelLsuTranspose,  // kModeTranspose: 6 CTAs/SM, 40 registers: 16 KiB tiles, more CTAs in different phases of the
                          // load -> shared -> store cycle (the fallback for transposes the tensor-map kernel cannot take)
    kKernelTransposeTma,  // kModeTransposeTma: tensor-map tile loads/stores around a register block transposition
                          // (transpose_tma.cu)
    kKernelCount
};

// The statistics buckets of tsnap_job_stats and tsnap_plan_info (bulk / rows / lsu), in launch order.
enum Bucket { kBucketBulk, kBucketRows, kBucketLsu, kBucketCount };

inline Kernel kernel_of(uint32_t mode) {
    switch (mode) {
        case kModeBulk: return kKernelBulk;
        case kModeRows: return kKernelRows;
        case kModeRowsTma: return kKernelRowsTma;
        case kModeStrided: return kKernelLsuStrided;
        case kModeTranspose: return kKernelLsuTranspose;
        case kModeTransposeTma: return kKernelTransposeTma;
        case kModeQChannel: return kKernelQChannel;
        case kModeQChannelFp8: return kKernelQChannelFp8;
        default: return kKernelLsu;  // kModeContig, kModeCast
    }
}
inline Bucket bucket_of(Kernel k) { return k == kKernelBulk ? kBucketBulk : k <= kKernelRowsTma ? kBucketRows : kBucketLsu; }

// one-time attribute setup (opt-in dynamic shared memory of the copy-engine kernels, occupancy of the LSU builds)
cudaError_t init_kernels();
// Launches kernel k over `ntiles` tiles of the device tables on `stream` (nothing when ntiles is 0): a persistent grid of
// the SM count times the kernel's resident CTAs per SM, capped at the tile count.  d_maps: the wave's tensor maps.
cudaError_t launch_kernel(Kernel k, const Member* d_members, const Tile* d_tiles, const TmaPair* d_maps, uint32_t ntiles,
                          int sm_count, cudaStream_t stream);

// launch_kernel for the kModeQChannel / kModeQChannelFp8 kernels (kKernelQStats .. kKernelQChannelFp8): `d_qch` is the wave's QChannel table, `nonfinite` a word the
// parameter kernel sets when a channel holds a NaN or Inf
cudaError_t launch_qchannel_kernel(Kernel k, const Member* d_members, const QChannel* d_qch, const Tile* d_tiles, uint32_t ntiles,
                                   int* nonfinite, int sm_count, cudaStream_t stream);

// transpose_tma.cu.  make_tma_pair encodes the two tensor maps of a kModeTranspose member (false: the member stays on the
// LSU transpose — 1-byte elements, bases or strides that are not 16 B multiples, more than 3 extra dims,
// TSNAP_B200_TMA_TRANSPOSE=0, or a driver without cuTensorMapEncodeTiled).
bool transpose_tma_enabled();
bool make_tma_pair(const Member& m, TmaPair* out, uint32_t* variant);  // variant = tile shape, for Member.shift bits 16-17
// kModeRowsTma: the same for kModeRows members with runs <= 1 KiB (TSNAP_B200_TMA_ROWS=0 keeps them on the per-run kernel)
bool make_rows_tma_pair(const Member& m, TmaPair* out);
cudaError_t init_transpose_tma();  // both tensor-map kernels
// launch_kernel for kKernelRowsTma and kKernelTransposeTma
cudaError_t launch_tma_kernel(Kernel k, const Member* d_members, const Tile* d_tiles, const TmaPair* d_maps, uint32_t ntiles,
                              int sm_count, cudaStream_t stream);
}  // namespace tsnap
