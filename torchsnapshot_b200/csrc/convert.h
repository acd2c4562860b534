// Element rules of the converting and quantising copies, bit for bit as torch converts: one definition for the host
// executor (plan.cpp) and the copy kernels (kernels.cu).  Where torch's CPU and CUDA results differ, a function keeps
// both behind __CUDA_ARCH__, the host executor giving the CPU's and the kernels the GPU's.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#ifdef __CUDACC__
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#endif

#include "../../include/tsnap_b200.h"

// host + device functions in a .cu translation unit, host functions in a .cpp one
#ifdef __CUDACC__
#define TSNAP_HD __host__ __device__ __forceinline__
#else
#define TSNAP_HD inline
#endif

namespace tsnap {

// ---- float8 ----------------------------------------------------------------------------------------------------------
// torch.float8_e4m3fn / torch.float8_e5m2 <-> fp32 (c10::Float8_e4m3fn and c10::Float8_e5m2 are built from a float and
// widen to a float, on the CPU and on the GPU alike).
//
//   narrowing: round to nearest even, subnormals kept.  e4m3fn has no infinity: values past 464 (the tie between 448,
//              its largest finite value, and the NaN pattern), +-inf and NaN all give 0x7F with the sign kept.  e5m2
//              overflows to +-inf (0x7C) from 61440 (the tie above 57344) on; NaN gives 0x7F with the sign kept.
//   widening:  exact.  An e4m3fn NaN becomes 0x7FF00000 (with its sign).  An e5m2 NaN becomes 0x7FFFFFFF on the
//              device, as torch's CUDA copy gives it, and keeps its payload on the host (torch's CPU loops differ there).
//
// Integer rounding rather than Hopper's cvt.rn.satfinite.{e4m3x2,e5m2x2}.f32: that instruction clamps overflow and
// infinities to the largest finite value, which is not torch's result.

TSNAP_HD uint32_t f32_bits(float f) {
    uint32_t u;
    std::memcpy(&u, &f, 4);
    return u;
}
TSNAP_HD float f32_from_bits(uint32_t u) {
    float f;
    std::memcpy(&f, &u, 4);
    return f;
}

// Below the smallest normal the value is added to 2^kMagic, whose fp32 ulp is the format's smallest subnormal: the
// fp32 adder rounds to nearest even at that ulp, and the low bits of the sum count subnormal steps (the count that
// reaches the smallest normal is its encoding as well).  Above it the fp32 exponent is rebiased and the 20 (e4m3fn)
// or 21 (e5m2) dropped mantissa bits are rounded to nearest even by integer addition.
TSNAP_HD uint8_t fp8_e4m3fn_from_f32(float f) {
    uint32_t u = f32_bits(f);
    const uint32_t sign = (u >> 24) & 0x80u;
    u &= 0x7FFFFFFFu;
    uint32_t r;
    if (u > 0x43E80000u) r = 0x7Fu;  // > 464, inf, NaN
    else if (u < 0x3C800000u) r = f32_bits(f32_from_bits(u) + 16384.0f) - 0x46800000u;  // < 2^-6: steps of 2^-9
    else r = (u - 0x3C000000u + 0x7FFFFu + ((u >> 20) & 1u)) >> 20;  // exponent bias 127 -> 7
    return uint8_t(r | sign);
}

TSNAP_HD uint8_t fp8_e5m2_from_f32(float f) {
    uint32_t u = f32_bits(f);
    const uint32_t sign = (u >> 24) & 0x80u;
    u &= 0x7FFFFFFFu;
    uint32_t r;
    if (u >= 0x47800000u) r = u > 0x7F800000u ? 0x7Fu : 0x7Cu;  // >= 65536: NaN stays NaN, the rest is inf
    else if (u < 0x38800000u) r = f32_bits(f32_from_bits(u) + 128.0f) - 0x43000000u;  // < 2^-14: steps of 2^-16
    else r = (u - 0x38000000u + 0xFFFFFu + ((u >> 21) & 1u)) >> 21;  // exponent bias 127 -> 15 (rounds up to inf at 61440)
    return uint8_t(r | sign);
}

TSNAP_HD float fp8_e4m3fn_to_f32(uint8_t b) {
    const uint32_t sign = uint32_t(b & 0x80u) << 24, e = (b >> 3) & 15u, m = b & 7u;
    if (e == 0) return f32_from_bits(f32_bits(float(m) * 0x1p-9f) | sign);  // zero and subnormals
    if (e == 15 && m == 7) return f32_from_bits(sign | 0x7FF00000u);
    return f32_from_bits(sign | ((e + 120u) << 23) | (m << 20));
}

TSNAP_HD float fp8_e5m2_to_f32(uint8_t b) {
    const uint32_t sign = uint32_t(b & 0x80u) << 24, e = (b >> 2) & 31u, m = b & 3u;
    if (e == 0) return f32_from_bits(f32_bits(float(m) * 0x1p-16f) | sign);  // zero and subnormals
    if (e == 31) {
#ifdef __CUDA_ARCH__
        if (m) return f32_from_bits(sign | 0x7FFFFFFFu);  // on the device torch's NaN is the canonical 0x7FFFFFFF
#endif
        return f32_from_bits(sign | 0x7F800000u | (m << 21));  // inf; on the host NaN keeps its payload
    }
    return f32_from_bits(sign | ((e + 112u) << 23) | (m << 21));
}

TSNAP_HD bool is_fp8_dtype(uint32_t dt) { return dt == TSNAP_F8E4M3FN || dt == TSNAP_F8E5M2; }

TSNAP_HD uint8_t fp8_from_f32(float f, uint32_t dt) { return dt == TSNAP_F8E4M3FN ? fp8_e4m3fn_from_f32(f) : fp8_e5m2_from_f32(f); }

TSNAP_HD float fp8_to_f32(uint8_t b, uint32_t dt) { return dt == TSNAP_F8E4M3FN ? fp8_e4m3fn_to_f32(b) : fp8_e5m2_to_f32(b); }

// ---- per-channel scaled float8 ---------------------------------------------------------------------------------------
// Largest finite value of each format.  An element x (as fp32) of a channel with scale s is stored as
// float8(clamp(x / s, -FMAX, FMAX)) with an IEEE fp32 division, and restored as fp32(q) * s in fp32.
TSNAP_HD float fp8_max(uint32_t dt) { return dt == TSNAP_F8E4M3FN ? 448.0f : 57344.0f; }
TSNAP_HD uint8_t fp8_quantize(float x, float s, uint32_t dt) {
    const float fmax = fp8_max(dt);
#ifdef __CUDA_ARCH__
    float y = __fdiv_rn(x, s);
#else
    float y = x / s;
#endif
    y = y < -fmax ? -fmax : (y > fmax ? fmax : y);
    return fp8_from_f32(y, dt);
}
TSNAP_HD float fp8_dequantize(uint8_t q, uint32_t dt, float s) { return fp8_to_f32(q, dt) * s; }

// ---- fp16 / bf16 <-> fp32 --------------------------------------------------------------------------------------------
// Widening is exact (a signalling NaN keeps its bits); narrowing rounds to nearest even and keeps subnormals.
TSNAP_HD float f16_to_f32(uint16_t h) {
#ifdef __CUDA_ARCH__
    return __half2float(__ushort_as_half(h));
#else
    _Float16 x;
    std::memcpy(&x, &h, 2);
    return float(x);
#endif
}
TSNAP_HD uint16_t f16_from_f32(float f) {
#ifdef __CUDA_ARCH__
    return __half_as_ushort(__float2half_rn(f));
#else
    const _Float16 x = (_Float16)f;
    uint16_t h;
    std::memcpy(&h, &x, 2);
    return h;
#endif
}
TSNAP_HD float bf16_to_f32(uint16_t v) {
#ifdef __CUDA_ARCH__
    return __bfloat162float(__ushort_as_bfloat16(v));
#else
    return f32_from_bits(uint32_t(v) << 16);
#endif
}
// c10::BFloat16's rounding.  A NaN gives what __float2bfloat16_rn gives on the device, as torch's CUDA copy does, and
// 0x7FC0 on the host: torch's CPU path has no fixed NaN encoding there (fp32 -> bf16 writes 0xFFFF, fp64 -> bf16 0x7FC0
// or 0xFFFF depending on whether its scalar or its vectorised loop ran).
TSNAP_HD uint16_t bf16_from_f32(float f) {
#ifdef __CUDA_ARCH__
    return __bfloat16_as_ushort(__float2bfloat16_rn(f));
#else
    if (std::isnan(f)) return 0x7FC0;
    const uint32_t u = f32_bits(f);
    return uint16_t((u + ((u >> 16) & 1) + 0x7FFFu) >> 16);
#endif
}
// fp32 -> a 2-byte float (TSNAP_F16 or TSNAP_BF16)
TSNAP_HD uint16_t f16_or_bf16_from_f32(float f, uint32_t dt) { return dt == TSNAP_BF16 ? bf16_from_f32(f) : f16_from_f32(f); }

// ---- elements at any alignment ---------------------------------------------------------------------------------------
// The n (2, 4 or 8) bytes of an element, little-endian; byte by byte unless `aligned` (a wire member behind an odd-sized
// one in an unpadded slab is not element aligned).
TSNAP_HD uint64_t load_bits(const char* p, uint32_t n, bool aligned) {
    if (aligned) return n == 8 ? *reinterpret_cast<const uint64_t*>(p) : n == 4 ? *reinterpret_cast<const uint32_t*>(p) : *reinterpret_cast<const uint16_t*>(p);
    uint64_t v = 0;
    for (int i = (int)n - 1; i >= 0; --i) v = (v << 8) | (uint8_t)p[i];
    return v;
}
TSNAP_HD void store_bytes(char* p, const void* v, int n, bool aligned) {
    const char* c = reinterpret_cast<const char*>(v);
    if (aligned) {
        if (n == 2) *reinterpret_cast<uint16_t*>(p) = *reinterpret_cast<const uint16_t*>(c);
        else if (n == 4) *reinterpret_cast<uint32_t*>(p) = *reinterpret_cast<const uint32_t*>(c);
        else *reinterpret_cast<uint64_t*>(p) = *reinterpret_cast<const uint64_t*>(c);
    } else {
        for (int i = 0; i < n; ++i) p[i] = c[i];
    }
}

// A wide float element (fp16, bf16, fp32, fp64) as fp32: fp64 rounds once, the others widen exactly.
TSNAP_HD float load_f32(const char* p, uint32_t dt, bool aligned) {
    switch (dt) {
        case TSNAP_F16: return f16_to_f32((uint16_t)load_bits(p, 2, aligned));
        case TSNAP_BF16: return bf16_to_f32((uint16_t)load_bits(p, 2, aligned));
        case TSNAP_F32: return f32_from_bits((uint32_t)load_bits(p, 4, aligned));
        default: {
            const uint64_t b = load_bits(p, 8, aligned);
            double x;
            std::memcpy(&x, &b, 8);
            return (float)x;
        }
    }
}
// An fp32 value as an element of float type dt: fp32 and fp64 exactly, fp16, bf16 and float8 rounded.
TSNAP_HD void store_f32(char* p, uint32_t dt, float f, bool aligned) {
    if (dt == TSNAP_F32) store_bytes(p, &f, 4, aligned);
    else if (dt == TSNAP_F16 || dt == TSNAP_BF16) { const uint16_t h = f16_or_bf16_from_f32(f, dt); store_bytes(p, &h, 2, aligned); }
    else if (is_fp8_dtype(dt)) *reinterpret_cast<uint8_t*>(p) = fp8_from_f32(f, dt);
    else { const double x = (double)f; store_bytes(p, &x, 8, aligned); }
}

// One element of a converting copy between two different float types, through fp32 as torch's copy kernel converts:
// sources of at most 32 bits widen exactly, with no detour through double (that would quiet the signalling NaNs torch's
// bf16 -> fp32 widening keeps bit for bit).  An fp64 source rounds once to fp32 and, for a narrower destination, once
// more: torch has no direct double -> half, bfloat16 or float8 conversion (c10::Half, c10::BFloat16 and c10::Float8_*
// are built from a float).  Float8 elements are single bytes: never misaligned.
TSNAP_HD void convert_store(char* p, uint32_t ddt, const char* sp, uint32_t sdt, bool src_aligned, bool aligned) {
    store_f32(p, ddt, is_fp8_dtype(sdt) ? fp8_to_f32(*reinterpret_cast<const uint8_t*>(sp), sdt) : load_f32(sp, sdt, src_aligned), aligned);
}

// ---- affine quantisation ---------------------------------------------------------------------------------------------
// torch's per-tensor quantize_val, clamped to the integer range.  ATen CPU (non-FBGEMM build) computes
// zero_point + nearbyint(x * (1.0f / scale)) in float, ATen CUDA (ATen/native/quantized/cuda/AffineQuantizer.cu)
// nearbyint(x / scale) + zero_point in double.
TSNAP_HD uint8_t quantize_elem(float x, double scale, int64_t zp, bool is_signed) {
#ifdef __CUDA_ARCH__
    long long q = (long long)(nearbyint((double)x / scale) + (double)zp);
#else
    long long q = zp + (long long)std::nearbyint(x * (1.0f / float(scale)));
#endif
    const long long lo = is_signed ? -128 : 0, hi = is_signed ? 127 : 255;
    q = q < lo ? lo : (q > hi ? hi : q);
    return (uint8_t)(int8_t)q;
}
// A quantised element back as fp32: float((q - zero_point) * scale), the product in double; store_f32 narrows it.
TSNAP_HD float dequantize(uint8_t raw, bool is_signed, int64_t zp, double scale) {
    const int64_t v = is_signed ? (int64_t)(int8_t)raw : (int64_t)raw;
    return (float)((double)(v - zp) * scale);
}

}  // namespace tsnap
