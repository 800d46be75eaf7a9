// fpng_b200/csrc/unfilter.cuh -- the per-row work of the unfilter kernels (D3: unfilter_kernel in decode_kernels.cu, writing uint8
// pixels, and unfilter_typed_kernel in decode_typed_kernels.cu, writing float32 / float16 / bfloat16): one thread per group of 4
// pixels loads its delta rows, runs the inverse Up filter (running sum down the columns) and converts 24 <-> 32 bpp.
#pragma once
#include "common.cuh"

namespace fpngb {

__device__ __forceinline__ uint32_t vadd4(uint32_t a, uint32_t b)
{
    const uint32_t s = (a & 0x7F7F7F7Fu) + (b & 0x7F7F7F7Fu);
    return s ^ ((a ^ b) & 0x80808080u);
}


// Delta rows y0 .. y0 + R - 1 (clamped to the last row) of a thread's group of npx pixels at delta: SRC words per row, the bytes
// past npx pixels zero.  R independent loads in flight per thread.
template <int SRC, int R>
__device__ __forceinline__ void load_delta_rows(const uint8_t* delta, uint32_t pitch, uint32_t y0, uint32_t h, bool full, uint32_t npx,
                                                uint32_t (&dd)[R][SRC])
{
#pragma unroll
    for (int j = 0; j < R; j++) {
        const uint32_t y = min(y0 + j, h - 1);
        const uint8_t* dr = delta + (size_t)y * pitch;
        if (full) {
#pragma unroll
            for (int i = 0; i < SRC; i++) dd[j][i] = __ldg(reinterpret_cast<const uint32_t*>(dr + 4 * i));   // pitch % 16 == 0 and x0*SRC % 4 == 0
        } else {
#pragma unroll
            for (int i = 0; i < SRC; i++) { dd[j][i] = 0; for (int b = 0; b < 4; b++) if ((uint32_t)(4 * i + b) < npx * SRC) dd[j][i] |= (uint32_t)dr[4 * i + b] << (8 * b); }
        }
    }
}

// One row of a group: the running sum of the delta words (a stored file's bytes are final as they are), then the 4 pixels
// repacked to DST interleaved channels in o[].
template <int SRC, int DST>
__device__ __forceinline__ void unfilter_row(uint32_t (&acc)[SRC], const uint32_t (&d)[SRC], bool summing, uint32_t (&o)[DST])
{
#pragma unroll
    for (int i = 0; i < SRC; i++) acc[i] = summing ? vadd4(acc[i], d[i]) : d[i];
    if (SRC == DST) {
#pragma unroll
        for (int i = 0; i < DST; i++) o[i] = acc[i];
    } else if (SRC == 3) {   // 24 -> 32 bpp, alpha 0xFF (fpng.cpp:2331)
        o[0] = (acc[0] & 0x00FFFFFFu) | 0xFF000000u;
        o[1] = __byte_perm(acc[0], acc[1], 0x4543) | 0xFF000000u;
        o[2] = __byte_perm(acc[1], acc[2], 0x4432) | 0xFF000000u;
        o[DST - 1] = (acc[2] >> 8) | 0xFF000000u;
    } else {                 // 32 -> 24 bpp, alpha dropped (fpng.cpp:2684-2721)
        o[0] = __byte_perm(acc[0], acc[1], 0x4210);
        o[1] = __byte_perm(acc[1], acc[2], 0x5421);
        o[DST - 1] = __byte_perm(acc[2], acc[SRC - 1], 0x6542);
    }
}

}  // namespace fpngb
