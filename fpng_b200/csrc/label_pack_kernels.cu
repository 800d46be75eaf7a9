// fpng_b200/csrc/label_pack_kernels.cu -- sm_90a pre-pass of fpngb_encode_label_ragged_device: reads each class id of every label
// map of the call once, checks its range and packs the ids into the PNG row bytes of the file (DESIGN §4.6, "Label maps"), which
// the PNG row kernels then encode as a gray8 image ceil(w * depth / 8) bytes wide, or as a gray16 image.
//
// One thread makes one 32-bit word of one packed row: 32 / depth ids (2 at depth 16), read with 16-, 8- or 4-byte loads where the ids are
// contiguous and aligned, one by one otherwise.  A CTA belongs to one image, so a warp flags an out-of-range id with one atomic.
#include "kernels.cuh"

namespace fpngb {

constexpr uint32_t kLabelThreads = 256;

uint32_t label_pack_ctas(uint32_t words, uint32_t h)
{
    return (uint32_t)(((unsigned long long)words * h + kLabelThreads - 1) / kLabelThreads);
}

// The output word of ids x0 .. x0 + PER - 1 of a row (ids past w are zero): depth D < 16 packs id j at bit 8 * byte + 8 - D - off
// of the little-endian word, (byte, off) = divmod(j * D, 8), i.e. MSB-first within each byte; D = 16 stores id j as the uint16 j.
template <class T, int D>
__device__ __forceinline__ uint32_t label_word(const uint8_t* q, unsigned long long pixel, uint32_t x0, uint32_t w, uint32_t limit, bool& bad)
{
    constexpr int PER = D == 16 ? 2 : 32 / D, RUN = PER * (int)sizeof(T);
    constexpr uint32_t mask = D == 16 ? 0xFFFFu : (1u << D) - 1u;
    uint32_t word = 0;
    auto put = [&](int j, unsigned long long v) {                           // v: the id as unsigned (a negative int64 is huge)
        bad |= v >= limit;
        const uint32_t f = (uint32_t)v & mask;
        if (D == 16) word |= f << (16 * j);
        else word |= f << (8 * ((j * D) >> 3) + 8 - D - ((j * D) & 7));
    };
    if (pixel == sizeof(T) && x0 + PER <= w && ((uintptr_t)q & (RUN >= 16 ? 15u : (uint32_t)RUN - 1u)) == 0) {
        if constexpr (RUN >= 16) {
#pragma unroll
            for (int i = 0; i < RUN / 16; i++) {
                const uint4 v = __ldg(reinterpret_cast<const uint4*>(q) + i);
                const uint32_t wd[4] = {v.x, v.y, v.z, v.w};
                if constexpr (sizeof(T) == 1) {
#pragma unroll
                    for (int b = 0; b < 16; b++) put(16 * i + b, (wd[b >> 2] >> (8 * (b & 3))) & 0xFFu);
                } else {
#pragma unroll
                    for (int e = 0; e < 2; e++) put(2 * i + e, ((unsigned long long)wd[2 * e + 1] << 32) | wd[2 * e]);
                }
            }
        } else {                                                            // uint8 ids at depth 4 (one 8-byte load) or 8 (4 bytes)
            uint32_t wd[2] = {0u, 0u};
            if constexpr (RUN == 8) { const uint2 v = __ldg(reinterpret_cast<const uint2*>(q)); wd[0] = v.x; wd[1] = v.y; }
            else wd[0] = __ldg(reinterpret_cast<const uint32_t*>(q));
#pragma unroll
            for (int b = 0; b < PER; b++) put(b, (wd[b >> 2] >> (8 * (b & 3))) & 0xFFu);
        }
    } else {
#pragma unroll 4
        for (int j = 0; j < PER; j++)
            if (x0 + j < w) put(j, (unsigned long long)(long long)__ldg(reinterpret_cast<const T*>(q + (unsigned long long)j * pixel)));
    }
    return word;
}

template <class T>
__device__ __forceinline__ uint32_t label_word_at(const LabelDesc& d, const uint8_t* q, uint32_t x0, bool& bad)
{
    switch (d.depth) {
    case 1: return label_word<T, 1>(q, d.pixel, x0, d.w, d.limit, bad);
    case 2: return label_word<T, 2>(q, d.pixel, x0, d.w, d.limit, bad);
    case 4: return label_word<T, 4>(q, d.pixel, x0, d.w, d.limit, bad);
    case 8: return label_word<T, 8>(q, d.pixel, x0, d.w, d.limit, bad);
    default:
        if constexpr (sizeof(T) == 8) return label_word<T, 16>(q, d.pixel, x0, d.w, d.limit, bad);
        else return 0u;                                                     // not reached: uint8 ids take depth <= 8
    }
}

__global__ void __launch_bounds__(kLabelThreads) label_pack_kernel(LabelPackParams p)
{
    uint32_t lo = 0, hi = p.count - 1;
    const unsigned long long b = blockIdx.x;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (p.desc[mid].cta_start <= b) lo = mid; else hi = mid - 1;
    }
    const LabelDesc& d = p.desc[lo];
    const unsigned long long g = (b - d.cta_start) * kLabelThreads + threadIdx.x;     // output word of the image
    bool bad = false;
    if (g < (unsigned long long)d.words * d.h) {
        const uint32_t y = (uint32_t)(g / d.words), k = (uint32_t)(g - (unsigned long long)y * d.words);
        const uint32_t x0 = k * (d.depth == 16 ? 2u : 32u / d.depth);
        const uint8_t* q = d.src + (unsigned long long)y * d.row + (unsigned long long)x0 * d.pixel;
        const uint32_t v = d.elem == 1 ? label_word_at<uint8_t>(d, q, x0, bad) : label_word_at<long long>(d, q, x0, bad);
        reinterpret_cast<uint32_t*>(p.dst + d.dst + (unsigned long long)y * 4ull * d.words)[k] = v;
    }
    if (__any_sync(0xFFFFFFFFu, bad) && (threadIdx.x & 31u) == 0) atomicOr(&p.bad[d.index], 1u);
}

void launch_label_pack(const LabelPackParams& p, unsigned long long total_ctas, cudaStream_t s)
{
    label_pack_kernel<<<(uint32_t)total_ctas, kLabelThreads, 0, s>>>(p);
}

}  // namespace fpngb
