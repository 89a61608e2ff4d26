// The row maths of every fp8 kernel (kv_fp8.cu, kv_fp8_pipe.cu): one 128-element row of bf16
// shares one fp32 scale.  The loops that walk rows stay in the kernels; what a row turns into
// is decided here, once.  The contract (docs/kernels.md, "fp8 row contract"), with rn32 f32
// round-to-nearest-even:
//   A     = max |x_i| over the finite x_i (0 if none): NaN and inf do not take part
//   scale = A > 0 ? max(rn32(A * rn32(1/448)), 2^-126) : 1
//   inv   = rn32(1 / scale)
//   q_i   = an e4m3 NaN code if x_i is not finite, else e4m3_satfinite_rne(rn32(x_i * inv))
//   y_i   = bf16_rne(rn32(e4m3(q_i) * scale))
// The floor of 2^-126 keeps the scale a normal number and inv <= 2^126: without it a row whose
// maximum is below 448 / FLT_MAX has inv = inf, and its zeros become NaN (0 * inf).  Mapping
// inf to NaN (drop_inf8) keeps one infinite element from making inv = 0 and the row's scale
// inf, which read back as a row of NaN.
// There is no direct bf16<->e4m3 cvt on sm_90a: quantise via f32, dequantise via f16x2 (e4m3
// -> f16 is exact).
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstdint>

namespace istore::kernels::fp8row {

constexpr float kE4m3Max = 448.f;
constexpr float kMinScale = 1.17549435e-38f;  // 2^-126, the smallest normal f32

__device__ __forceinline__ uint16_t cvt_e4m3x2(float hi, float lo) {  // F2FP.SATFINITE.E4M3.F32
    uint16_t r;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
    return r;
}
__device__ __forceinline__ uint32_t cvt_f16x2_e4m3x2(uint16_t v) {  // F2FP.F16.E4M3.UNPACK_B
    uint32_t r;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"(v));
    return r;
}
__device__ __forceinline__ float2 bf16x2_to_f2(uint32_t v) {
    return make_float2(__uint_as_float(v << 16), __uint_as_float(v & 0xffff0000u));
}
__device__ __forceinline__ uint32_t f2_to_bf16x2(float lo, float hi) {
    const __nv_bfloat162 b = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&b);
}

// Lane hl of the half-warp that owns a row: its 8 bf16 elements (one 16-byte vector) as f32,
// and their |max|.  fmaxf leaves NaN out of the |max|; an infinite element makes it inf, and
// the kernel then redoes the row with drop_inf8 (rows that hold +-inf only).
__device__ __forceinline__ float load8(uint4 v, float2 (&f)[4]) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        f[j] = bf16x2_to_f2(w[j]);
        amax = fmaxf(amax, fmaxf(fabsf(f[j].x), fabsf(f[j].y)));
    }
    return amax;
}

// True when a row's reduced |max| is inf: the row holds +-inf.
__device__ __forceinline__ bool has_inf(float amax) { return amax > 3.40282347e38f; }

// A row that holds +-inf: every infinite element becomes NaN, so that fmaxf leaves it out of
// the row's |max| and the cvt stores the e4m3 NaN code (satfinite alone would store +-448).
// Returns the |max| of the 8 elements again.  Kept off the common path: a select per element
// on every row cost the local-pool gathered write several per cent.
__device__ __forceinline__ float drop_inf8(float2 (&f)[4]) {
    const float nan = __uint_as_float(0x7fffffffu);
    float amax = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (fabsf(f[j].x) > 3.40282347e38f) f[j].x = nan;
        if (fabsf(f[j].y) > 3.40282347e38f) f[j].y = nan;
        amax = fmaxf(amax, fmaxf(fabsf(f[j].x), fabsf(f[j].y)));
    }
    return amax;
}

// The row's scale from its |max| (already reduced over the row).
__device__ __forceinline__ float row_scale(float amax) {
    return amax > 0.f ? fmaxf(amax * (1.f / kE4m3Max), kMinScale) : 1.f;
}

// 8 elements times inv as 8 e4m3 bytes (one 8-byte store).
__device__ __forceinline__ uint2 quant8(const float2 (&f)[4], float inv) {
    uint2 out;
    out.x = uint32_t(cvt_e4m3x2(f[0].y * inv, f[0].x * inv)) |
            (uint32_t(cvt_e4m3x2(f[1].y * inv, f[1].x * inv)) << 16);
    out.y = uint32_t(cvt_e4m3x2(f[2].y * inv, f[2].x * inv)) |
            (uint32_t(cvt_e4m3x2(f[3].y * inv, f[3].x * inv)) << 16);
    return out;
}

// 8 e4m3 values (v) times the row's scale, as 8 bf16 (one 16-byte store).
__device__ __forceinline__ uint4 dequant8(uint2 v, float sc) {
    const uint32_t w[2] = {v.x, v.y};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const uint32_t h01 = cvt_f16x2_e4m3x2(uint16_t(w[j] & 0xffffu));
        const uint32_t h23 = cvt_f16x2_e4m3x2(uint16_t(w[j] >> 16));
        const float2 f01 = __half22float2(*reinterpret_cast<const __half2*>(&h01));
        const float2 f23 = __half22float2(*reinterpret_cast<const __half2*>(&h23));
        o[2 * j] = f2_to_bf16x2(f01.x * sc, f01.y * sc);
        o[2 * j + 1] = f2_to_bf16x2(f23.x * sc, f23.y * sc);
    }
    return make_uint4(o[0], o[1], o[2], o[3]);
}

}  // namespace istore::kernels::fp8row
