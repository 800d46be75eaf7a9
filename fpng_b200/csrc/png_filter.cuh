// fpng_b200/csrc/png_filter.cuh -- the PNG row filters on packed bytes, shared by the general-PNG unfilter kernels
// (png_unfilter_kernels.cu): unaligned loads and stores of up to 4 bytes of a row, and the inverse of filter types 0-4 on 4 bytes at
// a time with the SIMD video intrinsics.
#pragma once
#include <stdint.h>

namespace fpngb {

__device__ __forceinline__ uint32_t load_px(const uint8_t* a, uint32_t bpp)
{
    uint32_t v = a[0];
    if (bpp > 1) v |= (uint32_t)a[1] << 8;
    if (bpp > 2) v |= (uint32_t)a[2] << 16;
    if (bpp > 3) v |= (uint32_t)a[3] << 24;
    return v;
}
__device__ __forceinline__ void store_px(uint8_t* a, uint32_t v, uint32_t bpp)
{
    a[0] = (uint8_t)v;
    if (bpp > 1) a[1] = (uint8_t)(v >> 8);
    if (bpp > 2) a[2] = (uint8_t)(v >> 16);
    if (bpp > 3) a[3] = (uint8_t)(v >> 24);
}

// the raw pixel of filter type ft from the filtered pixel x, left a, above b, upper-left c (PNG spec 9.2 - 9.4), byte-wise mod 256
__device__ __forceinline__ uint32_t unfilter_px(uint32_t ft, uint32_t x, uint32_t a, uint32_t b, uint32_t c)
{
    switch (ft) {
    case 1: return __vadd4(x, a);
    case 2: return __vadd4(x, b);
    case 3: return __vadd4(x, (a & b) + (((a ^ b) >> 1) & 0x7F7F7F7Fu));     // floor((a + b) / 2)
    case 4: {
        const uint32_t pa = __vabsdiffu4(b, c), pb = __vabsdiffu4(a, c);
        const uint32_t same = ~(__vcmpgeu4(b, c) ^ __vcmpgeu4(a, c));       // b - c and a - c of one sign: pc = pa + pb >= both
        const uint32_t pc = same | __vabsdiffu4(pa, pb);
        const uint32_t sel_a = __vcmpleu4(pa, pb) & __vcmpleu4(pa, pc);
        const uint32_t sel_b = ~sel_a & __vcmpleu4(pb, pc);
        return __vadd4(x, (a & sel_a) | (b & sel_b) | (c & ~(sel_a | sel_b)));
    }
    default: return x;
    }
}

}  // namespace fpngb
