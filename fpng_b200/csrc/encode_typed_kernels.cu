// fpng_b200/csrc/encode_typed_kernels.cu -- the conversion pre-pass of the encode calls: strided input -> tight integer HWC rows.
//
// convert_pixels_kernel<T, LAYOUT, PNG> reads an [n, h, w, chans] batch of T in an interleaved or planar layout ("Pixel layouts"
// of include/fpng_b200.h, strides in bytes) and writes tight rows of OB-byte samples (pitch w * chans * OB) into a library buffer;
// the integer encode pipeline then runs on that buffer unchanged.  Three uses:
//  * the *_typed fpng encode calls (T = float, __half, __nv_bfloat16; 3 or 4 channels, OB = 1): every element becomes
//        q = cvt.rni.sat.u8.f32( __fadd_rn(__fmul_rn((float)x, scale[c]), bias[c]) )
//    -- two separately rounded fp32 operations, never an FMA, then one round-to-nearest-even conversion that clamps to [0, 255]
//    and maps NaN to 0 (PTX ISA, cvt: float-to-integer conversions saturate, NaN converts to 0);
//  * the typed PNG encode call (PNG = true: 1 to 4 channels, OB from ConvDesc::sample_bytes): the same rule, with
//    cvt.rni.sat.u16.f32 for 16-bit samples, stored as native little-endian uint16 (the PNG row kernels swap the bytes);
//  * the strided uint8 input of the single-pass encoder, which reads tight rows only:
//    T = uint8_t, a plain copy.
// Each thread converts a group of 4 pixels of one row with the widest loads the address allows (16, 8, then 4 bytes, single
// elements at row ends).  The CTAs of a launch cover one or more descriptors; a CTA finds its descriptor by a binary search over
// their CTA prefix, as ragged_locate does.  All input addressing is 64-bit.  The PNG call has its own instantiations, so that the
// wider run-time switch costs the fpng calls' kernels no registers.
#include "kernels.cuh"
#include "typed_store.cuh"
#include "../../include/fpng_b200.h"
#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace fpngb {

constexpr uint32_t kConvThreads = 256;

template <typename T> __device__ __forceinline__ float elem_to_float(uint32_t bits);
template <> __device__ __forceinline__ float elem_to_float<float>(uint32_t bits) { return __uint_as_float(bits); }
template <> __device__ __forceinline__ float elem_to_float<__half>(uint32_t bits) { return __half2float(__ushort_as_half((unsigned short)bits)); }
template <> __device__ __forceinline__ float elem_to_float<__nv_bfloat16>(uint32_t bits) { return __uint_as_float(bits << 16); }

// element bits -> the OB-byte sample the encoder reads
template <typename T, int OB>
__device__ __forceinline__ uint32_t quantize(uint32_t bits, float scale, float bias)
{
    if constexpr (sizeof(T) == 1) {
        return bits;
    } else {
        const float y = __fadd_rn(__fmul_rn(elem_to_float<T>(bits), scale), bias);
        if constexpr (OB == 1) return round_u8(y);
        else return typed_bits<uint16_t>(y);                               // cvt.rni.sat.u16.f32
    }
}

template <int ES>
__device__ __forceinline__ uint32_t load_elem(const uint8_t* a)
{
    if constexpr (ES == 1) return __ldg(a);
    else if constexpr (ES == 2) return __ldg(reinterpret_cast<const unsigned short*>(a));
    else return __ldg(reinterpret_cast<const unsigned int*>(a));
}

// NW contiguous 32-bit words at a, which is ES-aligned: the widest loads the address allows
template <int ES, int NW>
__device__ __forceinline__ void load_words(const uint8_t* a, uint32_t (&wd)[NW])
{
    const uint32_t mis = (uint32_t)((uintptr_t)a & 15u);
    if (mis == 0u) {
        constexpr int N16 = NW / 4 * 4;
#pragma unroll
        for (int k = 0; k < N16; k += 4) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(a + 4 * k));
            wd[k] = v.x; wd[k + 1] = v.y; wd[k + 2] = v.z; wd[k + 3] = v.w;
        }
        if constexpr (NW - N16 >= 2) {
            const uint2 v = __ldg(reinterpret_cast<const uint2*>(a + 4 * N16));
            wd[N16] = v.x; wd[N16 + 1] = v.y;
        }
        if constexpr (NW % 2) wd[NW - 1] = __ldg(reinterpret_cast<const unsigned int*>(a + 4 * (NW - 1)));
    } else if ((mis & 7u) == 0u) {
#pragma unroll
        for (int k = 0; k + 2 <= NW; k += 2) {
            const uint2 v = __ldg(reinterpret_cast<const uint2*>(a + 4 * k));
            wd[k] = v.x; wd[k + 1] = v.y;
        }
        if constexpr (NW % 2) wd[NW - 1] = __ldg(reinterpret_cast<const unsigned int*>(a + 4 * (NW - 1)));
    } else if ((mis & 3u) == 0u) {
#pragma unroll
        for (int k = 0; k < NW; k++) wd[k] = __ldg(reinterpret_cast<const unsigned int*>(a + 4 * k));
    } else {
#pragma unroll
        for (int k = 0; k < NW; k++) {
            uint32_t v = 0;
#pragma unroll
            for (int e = 0; e < 4 / ES; e++) v |= load_elem<ES>(a + 4 * k + ES * e) << (8 * ES * e);
            wd[k] = v;
        }
    }
}

// element k of words wd[] of ES-byte elements
template <int ES, int NW>
__device__ __forceinline__ uint32_t word_elem(const uint32_t (&wd)[NW], int k)
{
    if constexpr (ES == 4) return wd[k];
    else if constexpr (ES == 2) return (wd[k >> 1] >> (16 * (k & 1))) & 0xFFFFu;
    else return (wd[k >> 2] >> (8 * (k & 3))) & 0xFFu;
}

// NW words to a (any alignment): the widest stores the address allows
template <int NW>
__device__ __forceinline__ void store_words(uint8_t* a, const uint32_t (&wd)[NW])
{
    const uint32_t mis = (uint32_t)((uintptr_t)a & 15u);
    if (mis == 0u) {
        constexpr int N16 = NW / 4 * 4;
#pragma unroll
        for (int k = 0; k < N16; k += 4) *reinterpret_cast<uint4*>(a + 4 * k) = make_uint4(wd[k], wd[k + 1], wd[k + 2], wd[k + 3]);
        if constexpr (NW - N16 >= 2) *reinterpret_cast<uint2*>(a + 4 * N16) = make_uint2(wd[N16], wd[N16 + 1]);
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
        for (int k = 0; k < 4 * NW; k++) a[k] = (uint8_t)(wd[k >> 2] >> (8 * (k & 3)));
    }
}

// One group of up to 4 pixels (x0 .. x0 + npx - 1) of one row: src at pixel x0 of the row, dst at byte x0 * CH * OB of the tight row.
template <typename T, bool PLANAR, int CH, int OB>
__device__ __forceinline__ void convert_group(const uint8_t* src, unsigned long long chan, uint8_t* dst, uint32_t npx, const ConvertParams& p)
{
    constexpr int ES = sizeof(T);
    uint32_t q[4 * CH];                                                     // output samples, interleaved
    if (npx == 4) {
        if (PLANAR) {                                                       // 4 * ES contiguous bytes per plane
#pragma unroll
            for (int c = 0; c < CH; c++) {
                uint32_t wd[ES];
                load_words<ES>(src + c * chan, wd);
#pragma unroll
                for (int k = 0; k < 4; k++) q[k * CH + c] = quantize<T, OB>(word_elem<ES>(wd, k), p.scale[c], p.bias[c]);
            }
        } else {                                                            // 4 * CH * ES contiguous bytes
            uint32_t wd[CH * ES];
            load_words<ES>(src, wd);
#pragma unroll
            for (int k = 0; k < 4 * CH; k++) q[k] = quantize<T, OB>(word_elem<ES>(wd, k), p.scale[k % CH], p.bias[k % CH]);
        }
        uint32_t ow[CH * OB];
#pragma unroll
        for (int k = 0; k < CH * OB; k++) {
            if constexpr (OB == 1) ow[k] = q[4 * k] | (q[4 * k + 1] << 8) | (q[4 * k + 2] << 16) | (q[4 * k + 3] << 24);
            else ow[k] = q[2 * k] | (q[2 * k + 1] << 16);
        }
        store_words(dst, ow);
    } else {                                                                // row end: element by element
        for (uint32_t x = 0; x < npx; x++) {
#pragma unroll
            for (int c = 0; c < CH; c++) {
                const uint8_t* a = PLANAR ? src + (size_t)x * ES + c * chan : src + ((size_t)x * CH + c) * ES;
                const uint32_t v = quantize<T, OB>(load_elem<ES>(a), p.scale[c], p.bias[c]);
                if constexpr (OB == 1) dst[x * CH + c] = (uint8_t)v;
                else reinterpret_cast<uint16_t*>(dst)[x * CH + c] = (uint16_t)v;   // dst is even: even pitch, 16-byte aligned base
            }
        }
    }
}

// CTA b - d.cta_start of descriptor d: items (image, row, 4-pixel group) in that order, kConvThreads per CTA.
template <typename T, bool PLANAR, int CH, int OB = 1>
__device__ __forceinline__ void convert_cta(const ConvDesc& d, unsigned long long local, const ConvertParams& p)
{
    constexpr int ES = sizeof(T);
    const unsigned long long img = local / d.ctas_per_image;
    const unsigned long long item = (local - img * d.ctas_per_image) * kConvThreads + threadIdx.x;
    const uint32_t groups = (d.w + 3u) >> 2;
    if (item >= (unsigned long long)d.h * groups) return;
    const uint32_t y = (uint32_t)(item / groups), x0 = (uint32_t)(item - (unsigned long long)y * groups) * 4u;
    const uint8_t* src = d.src + img * d.image + (unsigned long long)y * d.row + (unsigned long long)x0 * (PLANAR ? ES : CH * ES);
    uint8_t* dst = p.dst + d.dst + (img * d.h + y) * ((unsigned long long)d.w * CH * OB) + (unsigned long long)x0 * CH * OB;
    convert_group<T, PLANAR, CH, OB>(src, d.chan, dst, min(4u, d.w - x0), p);
}

// the PNG call's descriptors: 1 to 4 channels, OB = d.sample_bytes; one channel has no planes, so it reads as interleaved rows
template <typename T, bool PLANAR, int OB>
__device__ __forceinline__ void convert_cta_png(const ConvDesc& d, unsigned long long local, const ConvertParams& p)
{
    switch (d.chans) {
    case 1: convert_cta<T, false, 1, OB>(d, local, p); break;
    case 2: convert_cta<T, PLANAR, 2, OB>(d, local, p); break;
    case 3: convert_cta<T, PLANAR, 3, OB>(d, local, p); break;
    default: convert_cta<T, PLANAR, 4, OB>(d, local, p); break;
    }
}

template <typename T, int LAYOUT, bool PNG>
__global__ void __launch_bounds__(kConvThreads) convert_pixels_kernel(ConvertParams p)
{
    for (unsigned long long b = blockIdx.x; b < p.total_ctas; b += gridDim.x) {
        uint32_t lo = 0;
        if (p.count > 1) {
            uint32_t hi = p.count - 1;
            while (lo < hi) {
                const uint32_t mid = (lo + hi + 1) >> 1;
                if (p.desc[mid].cta_start <= b) lo = mid; else hi = mid - 1;
            }
        }
        const ConvDesc d = p.count > 1 ? p.desc[lo] : p.one;             // by value: no local copy of the parameter block
        const unsigned long long local = b - d.cta_start;
        const bool planar = LAYOUT == kConvAny ? d.planar != 0 : LAYOUT == kConvPlanar;
        if constexpr (PNG) {
            if (d.sample_bytes == 2) { if (planar) convert_cta_png<T, true, 2>(d, local, p); else convert_cta_png<T, false, 2>(d, local, p); }
            else { if (planar) convert_cta_png<T, true, 1>(d, local, p); else convert_cta_png<T, false, 1>(d, local, p); }
        } else if (planar) { if (d.chans == 3) convert_cta<T, true, 3>(d, local, p); else convert_cta<T, true, 4>(d, local, p); }
        else { if (d.chans == 3) convert_cta<T, false, 3>(d, local, p); else convert_cta<T, false, 4>(d, local, p); }
    }
}

uint32_t convert_ctas_per_image(uint32_t w, uint32_t h)
{
    return (uint32_t)(((unsigned long long)h * ((w + 3u) >> 2) + kConvThreads - 1) / kConvThreads);
}

template <typename T, bool PNG>
static void launch_t(const ConvertParams& p, int layout, uint32_t grid, cudaStream_t s)
{
    if (layout == kConvInterleaved) convert_pixels_kernel<T, kConvInterleaved, PNG><<<grid, kConvThreads, 0, s>>>(p);
    else if (layout == kConvPlanar) convert_pixels_kernel<T, kConvPlanar, PNG><<<grid, kConvThreads, 0, s>>>(p);
    else convert_pixels_kernel<T, kConvAny, PNG><<<grid, kConvThreads, 0, s>>>(p);
}

template <bool PNG>
static void launch_float(const ConvertParams& p, uint32_t dtype, int layout, uint32_t grid, cudaStream_t s)
{
    if (dtype == FPNGB_DTYPE_FLOAT32) launch_t<float, PNG>(p, layout, grid, s);
    else if (dtype == FPNGB_DTYPE_FLOAT16) launch_t<__half, PNG>(p, layout, grid, s);
    else launch_t<__nv_bfloat16, PNG>(p, layout, grid, s);
}

void launch_convert_pixels(const ConvertParams& p, uint32_t dtype, int layout, bool png, cudaStream_t s)
{
    if (!p.total_ctas) return;
    const uint32_t grid = (uint32_t)(p.total_ctas < (1ull << 24) ? p.total_ctas : (1ull << 24));   // grid-stride beyond that
    if (dtype == 0) {                                                                                // uint8 copy
        if (layout == kConvPlanar) convert_pixels_kernel<uint8_t, kConvPlanar, false><<<grid, kConvThreads, 0, s>>>(p);
        else convert_pixels_kernel<uint8_t, kConvInterleaved, false><<<grid, kConvThreads, 0, s>>>(p);
    } else if (png) launch_float<true>(p, dtype, layout, grid, s);
    else launch_float<false>(p, dtype, layout, grid, s);
}

}  // namespace fpngb
