// fpng_b200/csrc/typed_store.cuh -- element conversion and the wide stores of the kernels that write typed pixels
// (unfilter_typed_kernel, png_unfilter_kernel, decode_resize_kernel), and the choice of their element type.
#pragma once
#include "../../include/fpng_b200.h"
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace fpngb {

// Calls f with a value of the element type of an output dtype: float, __half, __nv_bfloat16, uint16_t, or uint8_t for dtype 0.  A
// launcher whose kernel has fewer types guards the others with if constexpr.
template <typename F>
inline void with_out_type(uint32_t dtype, F&& f)
{
    if (dtype == FPNGB_DTYPE_FLOAT32) f(float{});
    else if (dtype == FPNGB_DTYPE_FLOAT16) f(__half{});
    else if (dtype == FPNGB_DTYPE_BFLOAT16) f(__nv_bfloat16{});
    else if (dtype == FPNGB_DTYPE_UINT16) f(uint16_t{});
    else f(uint8_t{});
}

// v rounded to nearest even and clamped to [0, 255], NaN to 0 (PTX ISA, cvt: float-to-integer conversions saturate, NaN
// converts to 0): the quantiser of the typed encode
__device__ __forceinline__ uint32_t round_u8(float v)
{
    unsigned short q;
    asm("cvt.rni.sat.u8.f32 %0, %1;" : "=h"(q) : "f"(v));
    return q;
}

// the bit pattern of v stored as T: round to nearest even (overflow to +-inf for the float types, as torch's .to())
template <typename T> __device__ __forceinline__ uint32_t typed_bits(float v);
template <> __device__ __forceinline__ uint32_t typed_bits<float>(float v) { return __float_as_uint(v); }
template <> __device__ __forceinline__ uint32_t typed_bits<__half>(float v) { return __half_as_ushort(__float2half_rn(v)); }
template <> __device__ __forceinline__ uint32_t typed_bits<__nv_bfloat16>(float v) { return __bfloat16_as_ushort(__float2bfloat16_rn(v)); }
template <> __device__ __forceinline__ uint32_t typed_bits<uint8_t>(float v) { return round_u8(v); }
// v rounded to nearest even and clamped to [0, 65535], NaN to 0: uint16 output of the native resized decode (FPNGB_RESIZE_NATIVE)
template <> __device__ __forceinline__ uint32_t typed_bits<uint16_t>(float v)
{
    unsigned short q;
    asm("cvt.rni.sat.u16.f32 %0, %1;" : "=h"(q) : "f"(v));
    return q;
}
// The luma of 8-bit or 16-bit R, G, B (Pillow's convert("L") for 8-bit values; 32 bits hold it for 16-bit samples)
__device__ __forceinline__ uint32_t luma(uint32_t r, uint32_t g, uint32_t b) { return (19595u * r + 38470u * g + 7471u * b + 0x8000u) >> 16; }

__device__ __forceinline__ void store_elem(uint8_t* a, uint32_t bits, int size)
{
    if (size == 4) *reinterpret_cast<uint32_t*>(a) = bits;
    else if (size == 2) *reinterpret_cast<uint16_t*>(a) = (uint16_t)bits;
    else *a = (uint8_t)bits;
}

// NE contiguous elements of T (bit patterns e[]) at a, which is sizeof(T)-aligned: the widest stores the address allows, 16, then 8,
// then 4 bytes, else single elements.  NE * sizeof(T) is a multiple of 4 for every group shape here (4 pixels x 3 or 4 channels
// interleaved, 4 values of one plane).
template <typename T, int NE>
__device__ __forceinline__ void store_elems(uint8_t* a, const uint32_t (&e)[NE])
{
    constexpr int ES = sizeof(T), NW = NE * ES / 4;
    static_assert(NE * ES % 4 == 0, "whole 4-byte words");
    uint32_t wd[NW];
#pragma unroll
    for (int k = 0; k < NW; k++) {
        if constexpr (ES == 4) wd[k] = e[k];
        else if constexpr (ES == 2) wd[k] = e[2 * k] | (e[2 * k + 1] << 16);
        else wd[k] = e[4 * k] | (e[4 * k + 1] << 8) | (e[4 * k + 2] << 16) | (e[4 * k + 3] << 24);
    }
    const uint32_t mis = (uint32_t)((uintptr_t)a & 15u);
    if (mis == 0u) {
#pragma unroll
        for (int k = 0; k + 4 <= NW; k += 4) *reinterpret_cast<uint4*>(a + 4 * k) = make_uint4(wd[k], wd[k + 1], wd[k + 2], wd[k + 3]);
        constexpr int R = NW & ~3;
        if constexpr (NW % 4 >= 2) *reinterpret_cast<uint2*>(a + 4 * R) = make_uint2(wd[R], wd[R + 1]);
        if constexpr (NW % 2) *reinterpret_cast<uint32_t*>(a + 4 * (NW - 1)) = wd[NW - 1];
    } else if ((mis & 7u) == 0u) {
#pragma unroll
        for (int k = 0; k + 2 <= NW; k += 2) *reinterpret_cast<uint2*>(a + 4 * k) = make_uint2(wd[k], wd[k + 1]);
        if constexpr (NW % 2) *reinterpret_cast<uint32_t*>(a + 4 * (NW - 1)) = wd[NW - 1];
    } else if ((mis & 3u) == 0u) {
#pragma unroll
        for (int k = 0; k < NW; k++) *reinterpret_cast<uint32_t*>(a + 4 * k) = wd[k];
    } else {
#pragma unroll
        for (int k = 0; k < NE; k++) store_elem(a + ES * k, e[k], ES);
    }
}

}  // namespace fpngb
