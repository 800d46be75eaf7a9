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
#include "typed_store.cuh"
#include "../../include/fpng_b200.h"

namespace fpngb {

void launch_png_inflate(const PngParams& p, cudaStream_t s);

constexpr uint32_t kUnfilterWarps = 4;

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
    const uint32_t w = fd.w, h = fd.h, bpp = fd.chans, D = p.desired, stride = w * bpp + 1u;
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
            if constexpr (ES == 1) {
                if (D == 4) *reinterpret_cast<uint32_t*>(po) = o;           // 16-byte aligned file, 4-byte pixels
                else { po[0] = (uint8_t)o; po[1] = (uint8_t)(o >> 8); po[2] = (uint8_t)(o >> 16); }
            } else {
#pragma unroll
                for (uint32_t k = 0; k < 4; k++) {
                    if (k >= D) break;
                    const float v = __uint2float_rn((o >> (8 * k)) & 0xFFu);
                    store_elem(po + k * ES, typed_bits<T>(__fadd_rn(__fmul_rn(v, pa.scale[k]), pa.bias[k])), ES);
                }
            }
        }
        __syncwarp();
    }
}

void launch_png_decode(const PngParams& p, const TypedOut* typed, cudaStream_t s)
{
    launch_png_inflate(p, s);
    const dim3 g((p.n + kUnfilterWarps - 1) / kUnfilterWarps), b(32 * kUnfilterWarps);
    const PixelAffine pa = typed ? typed->aff : PixelAffine{};
    if (!typed) png_unfilter_kernel<uint8_t><<<g, b, 0, s>>>(p, pa);
    else if (typed->dtype == FPNGB_DTYPE_FLOAT32) png_unfilter_kernel<float><<<g, b, 0, s>>>(p, pa);
    else if (typed->dtype == FPNGB_DTYPE_FLOAT16) png_unfilter_kernel<__half><<<g, b, 0, s>>>(p, pa);
    else png_unfilter_kernel<__nv_bfloat16><<<g, b, 0, s>>>(p, pa);
}

}  // namespace fpngb
