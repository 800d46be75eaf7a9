// fpng_b200/csrc/png_unfilter_kernels.cu -- unfilter and store of the general PNG files of the any-PNG decodes, and the launch
// sequence of their pipeline (gather, inflate: inflate_kernels.cu).
//
// Sub, Avg and Paeth chain along a row and Up, Avg and Paeth down the rows, so a file is a 2-D dependency.  png_unfilter_kernel runs
// it as a wavefront, one warp per file, 32 rows per band: lane k owns row y0 + k and runs k pixels behind lane k - 1.  At each step
// one __shfl_up_sync hands a lane the pixel above it (b, what lane k - 1 finished on the previous step); the value it received on
// the previous step is the up-left pixel (c); lane 0 reads the row above the band, which the band before wrote back in place.  A
// band takes w + 31 steps instead of 32 w.  The byte arithmetic runs on whole pixels, 4 bytes at a time, with the SIMD video
// intrinsics (Paeth included: |p - a| = |b - c|, |p - b| = |a - c|, and |p - c| is their sum when b - c and a - c have the same
// sign, else the absolute difference of the two).  Each pixel is expanded to the output channels (gray -> Y Y Y, alpha 255 when the
// file has none) and stored as uint8 or through typed_store.cuh's conversion into the ragged tight rows.  The kernel also writes every
// general file's final status to d_status: decode_status_kernel, earlier in the stream, wrote the internal kPngPending there.
#include "decode.cuh"
#include "png_filter.cuh"
#include "png_walk.cuh"
#include "typed_store.cuh"
#include "../../include/fpng_b200.h"
#include <type_traits>

namespace fpngb {

void launch_png_inflate(const PngParams& p, cudaStream_t s);

constexpr uint32_t kUnfilterWarps = 4;

// channel k (0..3) of the output pixel of raw file pixel v with bpp bytes: gray Y -> Y Y Y 255, gray+alpha -> Y Y Y A, RGB -> R G B 255
__device__ __forceinline__ uint32_t expand_px(uint32_t v, uint32_t bpp)
{
    if (bpp == 1) return (v & 0xFFu) * 0x010101u | 0xFF000000u;
    if (bpp == 2) return (v & 0xFFu) * 0x010101u | (v << 16 & 0xFF000000u);
    if (bpp == 3) return v | 0xFF000000u;
    return v;
}

template <typename T>
__global__ void __launch_bounds__(32 * kUnfilterWarps) png_unfilter_kernel(PngParams p, PixelAffine pa)
{
    constexpr uint32_t ES = sizeof(T);
    const uint32_t lane = threadIdx.x & 31u, f = blockIdx.x * kUnfilterWarps + (threadIdx.x >> 5);
    if (f >= p.n) return;
    const FileDesc fd = p.files[f];
    if (fd.pre_status != kPngPending) return;
    const uint32_t st = p.png[f].status;
    if (lane == 0) p.d_status[f] = st;
    if (st) return;
    const uint32_t w = fd.w, h = fd.h, bpp = fd.chans, D = p.desired ? p.desired : bpp, stride = w * bpp + 1u;
    uint8_t* rows = p.rows + fd.delta_base;
    uint8_t* out = p.d_out + fd.out_base;
    for (uint32_t y0 = 0; y0 < h; y0 += 32) {
        const uint32_t y = y0 + lane;
        const bool active = y < h;
        uint8_t* row = rows + (size_t)(active ? y : 0) * stride;
        const uint8_t* above = y0 ? rows + (size_t)(y0 - 1) * stride + 1 : nullptr;   // lane 0: raw, written back by the band before
        const uint32_t ft = active ? row[0] : 0u;
        const bool write_back = lane == 31 && y0 + 32 < h;
        uint8_t* orow = out + (size_t)(active ? y : 0) * w * D * ES;
        uint32_t a = 0, c = 0, cur = 0;
        for (uint32_t t = 0; t < w + 31; t++) {
            const uint32_t up = __shfl_up_sync(0xFFFFFFFFu, cur, 1);
            const int x = (int)t - (int)lane;
            if (!active || x < 0 || x >= (int)w) continue;
            const uint32_t b = lane ? up : (above ? load_px(above + (size_t)x * bpp, bpp) : 0u);
            const uint32_t raw = unfilter_px(ft, load_px(row + 1 + (size_t)x * bpp, bpp), a, b, c);
            c = b; a = raw; cur = raw;
            if (write_back) store_px(row + 1 + (size_t)x * bpp, raw, bpp);
            const uint32_t o = expand_px(raw, bpp);
            uint8_t* po = orow + (size_t)x * D * ES;
            if (ES == 1 && D == 4) { *reinterpret_cast<uint32_t*>(po) = o; continue; }   // 16-byte aligned file, 4-byte pixels
            // D 1 / 2: L or (L, A); gray's luma is Y itself
            const uint32_t l = D > 2 ? o : luma(o & 0xFFu, o >> 8 & 0xFFu, o >> 16 & 0xFFu) | (o >> 16 & 0xFF00u);
#pragma unroll
            for (uint32_t k = 0; k < 4; k++) {
                if (k >= D) break;
                const uint32_t v = (l >> (8 * k)) & 0xFFu;
                if constexpr (ES == 1) po[k] = (uint8_t)v;
                else if constexpr (std::is_same<T, uint16_t>::value) store_elem(po + k * ES, p.index ? v : v * 257u, ES);
                else store_elem(po + k * ES, typed_bits<T>(__fadd_rn(__fmul_rn(__uint2float_rn(v), pa.scale[k]), pa.bias[k])), ES);
            }
        }
        __syncwarp();
    }
}

// ---- the other formats (FPNGB_PNG_ALL_FORMATS): palette, 1/2/4/16-bit, color keys, Adam7 --------------------------------------
// png_unfilter_ext_kernel: one warp per ext file (pre_status kPngPendingExt).  It first checks the filter byte of every row of every
// pass, so that a bad one gives FAILED_INVALID_IDAT before any pixel is written (and before the inflate's Adler-32 mismatch, the
// order the 8-bit files get), then writes the file's final status.  Palette files stage their 256 entries, tRNS alpha folded in and
// (0, 0, 0, 255) past the entry count, as packed RGBA words in shared memory.  Each pass (one for interlace 0, Adam7's seven) runs
// png_unfilter_kernel's wavefront over filter units of max(1, bits_per_pixel / 8) bytes, held in two words (lo: bytes 0-3, hi: bytes
// 4-7) with the same byte arithmetic.  A unit expands to one pixel, or 8 / depth pixels for the sub-byte depths (padding bits past
// the pass width ignored), each placed at its image position (x0 + i dx, y0 + j dy).  Pixels are carried as four 16-bit channels:
// 16-bit samples as they are, 8-bit values v (palette entries and scaled gray included) as v * 257, an alpha the file does not
// have and a color key's 0 / 255 as 0 / 0xFFFF.  uint8 output stores the high bytes; typed output converts v = s / 257 for 16-bit
// files (the header's rule) and v = s >> 8 otherwise.  An index call (PngParams::index) stages no palette and stores each pixel's
// raw sample (palette index, gray sample of any depth) as it is, through store_index.
// The launch bound's 4 CTAs per SM allow up to 128 registers: without it ptxas kept this kernel at 64 and spilled.
constexpr uint32_t kExtWarps = 4;

// channel value s (16-bit domain) of a file of depth 16 (wide) or below as the float the typed conversion starts from
__device__ __forceinline__ float ext_value(uint32_t s, bool wide)
{
    return wide ? __fdiv_rn(__uint2float_rn(s), 257.0f) : __uint2float_rn(s >> 8);
}

// one output pixel: rg = R | G << 16, ba = B | A << 16 in the 16-bit domain
template <typename T>
__device__ __forceinline__ void store_ext_px(uint8_t* po, uint32_t rg, uint32_t ba, uint32_t D, bool wide, const PixelAffine& pa)
{
    constexpr uint32_t ES = sizeof(T);
    if (ES == 1 && D >= 3) {                                                // uint8 at D 3 / 4: the high bytes
        const uint32_t o = (rg >> 8 & 0xFFu) | (rg >> 16 & 0xFF00u) | (ba << 8 & 0xFF0000u) | (ba & 0xFF000000u);
        if (D == 4) *reinterpret_cast<uint32_t*>(po) = o;                   // 16-byte aligned file, 4-byte pixels
        else { po[0] = (uint8_t)o; po[1] = (uint8_t)(o >> 8); po[2] = (uint8_t)(o >> 16); }
        return;
    }
    if (D <= 2) {                           // L or (L, A): L from 16-bit samples, or from the 8-bit values v = s >> 8 (then * 257)
        const uint32_t r = rg & 0xFFFFu, g = rg >> 16, b = ba & 0xFFFFu;
        const uint32_t l = wide ? luma(r, g, b) : luma(r >> 8, g >> 8, b >> 8) * 257u;
        rg = l | (ba & 0xFFFF0000u);        // channel 0 L, channel 1 A
    }
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) {
        if (k >= D) break;
        const uint32_t s = D <= 2 ? (rg >> (16 * k)) & 0xFFFFu : ((k < 2 ? rg : ba) >> (16 * (k & 1u))) & 0xFFFFu;
        if constexpr (ES == 1) po[k] = (uint8_t)(s >> 8);
        else if constexpr (std::is_same<T, uint16_t>::value) store_elem(po + k * ES, s, ES);
        else store_elem(po + k * ES, typed_bits<T>(__fadd_rn(__fmul_rn(ext_value(s, wide), pa.scale[k]), pa.bias[k])), ES);
    }
}

// the raw sample s of an index call: uint8 or uint16 output, desired 1 (the walk gave every file s does not fit FPNGB_DECODE_NOT_INDEXED)
template <typename T>
__device__ __forceinline__ void store_index(uint8_t* po, uint32_t s)
{
    if constexpr (sizeof(T) == 1 || std::is_same<T, uint16_t>::value) store_elem(po, s, sizeof(T));
}

__device__ __forceinline__ uint32_t unit_byte(uint32_t lo, uint32_t hi, uint32_t j) { return ((j < 4 ? lo : hi) >> (8 * (j & 3u))) & 0xFFu; }

template <typename T>
__global__ void __launch_bounds__(32 * kExtWarps, 4) png_unfilter_ext_kernel(PngParams p, PixelAffine pa)
{
    __shared__ uint32_t s_pal[kExtWarps][256];
    constexpr uint32_t ES = sizeof(T);
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, f = blockIdx.x * kExtWarps + warp;
    if (f >= p.n) return;
    const FileDesc fd = p.files[f];
    if (fd.pre_status != kPngPendingExt) return;
    const PngDesc pd = p.png[f];
    const uint32_t w = fd.w, h = fd.h, D = p.desired ? p.desired : fd.chans, depth = pd.depth, type = pd.type;
    const uint32_t passes = pd.interlace ? 7u : 1u;
    const uint32_t samples = type == 2 ? 3u : type == 4 ? 2u : type == 6 ? 4u : 1u;
    const uint32_t bits = depth * samples, U = bits < 8 ? 1u : bits / 8;
    const bool wide = depth == 16;
    uint8_t* rows = p.rows + fd.delta_base;
    uint32_t st = pd.status;
    if (st == 0 || st == FPNGB_DECODE_ADLER_MISMATCH) {                     // the stream inflated to raw_len bytes: filter bytes
        bool bad = false;
        unsigned long long at = 0;
        for (uint32_t k = 0; k < passes; k++) {
            uint32_t x0 = 0, y0 = 0, dx = 1, dy = 1;
            if (passes > 1) adam7_pass(k, &x0, &y0, &dx, &dy);
            const uint32_t pw = pass_extent(w, x0, dx), ph = pass_extent(h, y0, dy);
            if (!pw || !ph) continue;
            const unsigned long long stride = 1ull + ((unsigned long long)pw * bits + 7) / 8;
            for (uint32_t y = lane; y < ph; y += 32) bad |= rows[at + y * stride] > 4;
            at += ph * stride;
        }
        if (__any_sync(0xFFFFFFFFu, bad)) st = FPNGB_DECODE_FAILED_INVALID_IDAT;
    }
    if (lane == 0) p.d_status[f] = st;
    if (st) return;
    const uint8_t* file = p.d_files + fd.base;
    uint32_t* pal = s_pal[warp];
    if (type == 3 && !p.index) {
        for (uint32_t i = lane; i < 256; i += 32) {
            uint32_t e = 0xFF000000u;
            if (i < pd.plte_n) {
                const uint8_t* q = file + pd.plte_ofs + 3 * i;
                const uint32_t a = i < pd.trns_len ? file[pd.trns_ofs + i] : 255u;
                e = q[0] | (uint32_t)q[1] << 8 | (uint32_t)q[2] << 16 | a << 24;
            }
            pal[i] = e;
        }
        __syncwarp();
    }
    // color key (tRNS in types 0 / 2): full samples; 0x10000 + never matches a file without one
    uint32_t k0 = 0x10000u, k1 = 0x10000u, k2 = 0x10000u;
    if (pd.trns_ofs && (type == 0 || type == 2)) {
        const uint8_t* t = file + pd.trns_ofs;
        k0 = (uint32_t)t[0] << 8 | t[1];
        if (type == 2) { k1 = (uint32_t)t[2] << 8 | t[3]; k2 = (uint32_t)t[4] << 8 | t[5]; }
    }
    const uint32_t sub_mask = (1u << (depth < 8 ? depth : 1u)) - 1u, sub_per = depth < 8 ? 8 / depth : 1u;
    const uint32_t gray_mul = depth < 8 ? 255u / sub_mask * 257u : 257u;    // gray below 8 bits: s * 255 / (2^d - 1), then * 257
    uint8_t* out = p.d_out + fd.out_base;
    unsigned long long at = 0;
    for (uint32_t k = 0; k < passes; k++) {
        uint32_t x0 = 0, y0 = 0, dx = 1, dy = 1;
        if (passes > 1) adam7_pass(k, &x0, &y0, &dx, &dy);
        const uint32_t pw = pass_extent(w, x0, dx), ph = pass_extent(h, y0, dy);
        if (!pw || !ph) continue;
        const uint32_t rb = (uint32_t)(((unsigned long long)pw * bits + 7) / 8), stride = rb + 1u, nu = bits < 8 ? rb : pw;
        uint8_t* prow = rows + at;
        for (uint32_t b0 = 0; b0 < ph; b0 += 32) {
            const uint32_t py = b0 + lane;
            const bool active = py < ph;
            uint8_t* row = prow + (size_t)(active ? py : 0) * stride;
            const uint8_t* above = b0 ? prow + (size_t)(b0 - 1) * stride + 1 : nullptr;   // lane 0: raw, written back by the band before
            const uint32_t ft = active ? row[0] : 0u;
            const bool write_back = lane == 31 && b0 + 32 < ph;
            uint8_t* orow = out + (size_t)(active ? y0 + py * dy : 0) * w * D * ES;
            uint32_t alo = 0, ahi = 0, clo = 0, chi = 0, cur_lo = 0, cur_hi = 0;
            for (uint32_t t = 0; t < nu + 31; t++) {
                const uint32_t up_lo = __shfl_up_sync(0xFFFFFFFFu, cur_lo, 1);
                const uint32_t up_hi = U > 4 ? __shfl_up_sync(0xFFFFFFFFu, cur_hi, 1) : 0u;
                const int x = (int)t - (int)lane;
                if (!active || x < 0 || x >= (int)nu) continue;
                uint32_t blo = up_lo, bhi = up_hi;
                const uint8_t* src = row + 1 + (size_t)x * U;
                if (!lane) {
                    blo = above ? load_px(above + (size_t)x * U, U < 4 ? U : 4u) : 0u;
                    bhi = above && U > 4 ? load_px(above + (size_t)x * U + 4, U - 4) : 0u;
                }
                const uint32_t rlo = unfilter_px(ft, load_px(src, U < 4 ? U : 4u), alo, blo, clo);
                const uint32_t rhi = U > 4 ? unfilter_px(ft, load_px(src + 4, U - 4), ahi, bhi, chi) : 0u;
                clo = blo; chi = bhi; alo = cur_lo = rlo; ahi = cur_hi = rhi;
                if (write_back) { store_px(row + 1 + (size_t)x * U, rlo, U < 4 ? U : 4u); if (U > 4) store_px(row + 5 + (size_t)x * U, rhi, U - 4); }
                if (depth < 8) {                                            // 8 / depth pixels, most significant bits first
                    for (uint32_t j = 0; j < sub_per; j++) {
                        const uint32_t i = (uint32_t)x * sub_per + j;
                        if (i >= pw) break;
                        const uint32_t s = rlo >> (8 - depth * (j + 1)) & sub_mask;
                        if (p.index) { store_index<T>(orow + (size_t)(x0 + i * dx) * ES, s); continue; }
                        uint32_t rg, ba;
                        if (type == 3) {
                            const uint32_t e = pal[s];
                            rg = (e & 0xFFu) * 257u | (e >> 8 & 0xFFu) * 257u << 16;
                            ba = (e >> 16 & 0xFFu) * 257u | (e >> 24) * 257u << 16;
                        } else {
                            const uint32_t y = s * gray_mul;
                            rg = y | y << 16;
                            ba = y | (s == k0 ? 0u : 0xFFFF0000u);
                        }
                        store_ext_px<T>(orow + (size_t)(x0 + i * dx) * D * ES, rg, ba, D, false, pa);
                    }
                    continue;
                }
                // one pixel: its samples in the 16-bit domain, and the raw samples the color key compares
                uint32_t s[4];
#pragma unroll
                for (uint32_t m = 0; m < 4; m++)
                    s[m] = wide ? unit_byte(rlo, rhi, 2 * m) << 8 | unit_byte(rlo, rhi, 2 * m + 1) : unit_byte(rlo, rhi, m);
                if (p.index) { store_index<T>(orow + (size_t)(x0 + (uint32_t)x * dx) * ES, s[0]); continue; }
                uint32_t rg, ba;
                const uint32_t mul = wide ? 1u : 257u;
                if (type == 3) {
                    const uint32_t e = pal[s[0]];
                    rg = (e & 0xFFu) * 257u | (e >> 8 & 0xFFu) * 257u << 16;
                    ba = (e >> 16 & 0xFFu) * 257u | (e >> 24) * 257u << 16;
                } else if (type == 0 || type == 4) {
                    const uint32_t y = s[0] * mul;
                    const uint32_t a = type == 4 ? s[1] * mul : s[0] == k0 ? 0u : 0xFFFFu;
                    rg = y | y << 16; ba = y | a << 16;
                } else {
                    const uint32_t a = type == 6 ? s[3] * mul : (s[0] == k0 && s[1] == k1 && s[2] == k2) ? 0u : 0xFFFFu;
                    rg = s[0] * mul | s[1] * mul << 16; ba = s[2] * mul | a << 16;
                }
                store_ext_px<T>(orow + (size_t)(x0 + (uint32_t)x * dx) * D * ES, rg, ba, D, wide, pa);
            }
            __syncwarp();
        }
        at += (unsigned long long)ph * stride;
    }
}

void launch_png_decode(const PngParams& p, const TypedOut* typed, uint32_t flags, cudaStream_t s)
{
    launch_png_inflate(p, s);
    const PixelAffine pa = typed ? typed->aff : PixelAffine{};
    with_out_type(typed ? typed->dtype : 0u, [&](auto t) {
        using T = decltype(t);
        png_unfilter_kernel<T><<<(p.n + kUnfilterWarps - 1) / kUnfilterWarps, 32 * kUnfilterWarps, 0, s>>>(p, pa);
        if (flags & FPNGB_PNG_ALL_FORMATS) png_unfilter_ext_kernel<T><<<(p.n + kExtWarps - 1) / kExtWarps, 32 * kExtWarps, 0, s>>>(p, pa);
    });
}

}  // namespace fpngb
