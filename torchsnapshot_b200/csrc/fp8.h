// torch.float8_e4m3fn / torch.float8_e5m2 <-> fp32, bit for bit as torch converts them (c10::Float8_e4m3fn and
// c10::Float8_e5m2 are built from a float and widen to a float, on the CPU and on the GPU alike).  One definition for
// the host executor (plan.cpp) and the copy kernels (kernels.cu).
//
//   narrowing: round to nearest even, subnormals kept.  e4m3fn has no infinity: values past 464 (the tie between 448,
//              its largest finite value, and the NaN pattern), +-inf and NaN all give 0x7F with the sign kept.  e5m2
//              overflows to +-inf (0x7C) from 61440 (the tie above 57344) on; NaN gives 0x7F with the sign kept.
//   widening:  exact.  An e4m3fn NaN becomes 0x7FF00000 (with its sign).  An e5m2 NaN becomes 0x7FFFFFFF on the
//              device, as torch's CUDA copy gives it, and keeps its payload on the host (torch's CPU loops differ there).
//
// Integer rounding rather than Hopper's cvt.rn.satfinite.{e4m3x2,e5m2x2}.f32: that instruction clamps overflow and
// infinities to the largest finite value, which is not torch's result.  Callers convert wider and narrower sources
// through fp32, as torch does (an fp64 value is rounded twice).
#pragma once
#include <cstdint>
#include <cstring>

#include "../../include/tsnap_b200.h"

#ifdef __CUDACC__
#define TSNAP_HD __host__ __device__ __forceinline__
#else
#define TSNAP_HD inline
#endif

namespace tsnap {

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

}  // namespace tsnap
