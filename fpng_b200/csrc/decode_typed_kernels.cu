// fpng_b200/csrc/decode_typed_kernels.cu -- D3 typed: the unfilter pass of the *_typed decode calls (include/fpng_b200.h,
// fpngb_pixel_format).  unfilter_kernel's running sum (unfilter.cuh) with every value converted in registers and stored as float32,
// float16 or bfloat16: no uint8 buffer and no extra pass over the pixels.  v * scale + bias is two separately rounded fp32
// operations (never an FMA: what numpy and torch eager compute for x * s + b), then round to nearest even into T (overflow to
// +-inf, as torch's .to()).  Its own translation unit, so that the uint8 decode kernels compile exactly as they did.
#include "decode.cuh"
#include "unfilter.cuh"
#include "typed_store.cuh"
#include "../../include/fpng_b200.h"
#include <type_traits>

namespace fpngb {

// byte k of the interleaved pixel bytes o[] (k = pixel * DST + channel), mapped to channel c and converted; the native calls'
// uint8 and uint16 output (FPNGB_PNG_NATIVE) store the value v and v * 257, with no scale or bias
template <typename T, int DST>
__device__ __forceinline__ uint32_t typed_value(const uint32_t (&o)[DST], int k, int c, const PixelAffine& pa)
{
    const uint32_t b = (o[k >> 2] >> (8 * (k & 3))) & 0xFFu;
    if constexpr (sizeof(T) == 1) return b;
    else if constexpr (std::is_same<T, uint16_t>::value) return b * 257u;
    else return typed_bits<T>(__fadd_rn(__fmul_rn(__uint2float_rn(b), pa.scale[c]), pa.bias[c]));
}

// DST 1 / 2 (native calls): the 4 pixels of a group as L or (L, A) bytes, L the luma of R, G, B (typed_store.cuh), A 255 for SRC 3
template <int SRC, int DST>
__device__ __forceinline__ void luma_row(const uint32_t (&px)[SRC], uint32_t (&o)[DST])
{
#pragma unroll
    for (int i = 0; i < DST; i++) o[i] = 0;
#pragma unroll
    for (int q = 0; q < 4; q++) {
        const int k = q * SRC;
        const uint32_t r = (px[k >> 2] >> (8 * (k & 3))) & 0xFFu, g = (px[(k + 1) >> 2] >> (8 * ((k + 1) & 3))) & 0xFFu,
                       b = (px[(k + 2) >> 2] >> (8 * ((k + 2) & 3))) & 0xFFu;
        const uint32_t a = SRC == 4 ? (px[(k + 3) >> 2] >> (8 * ((k + 3) & 3))) & 0xFFu : 0xFFu;
        const uint32_t v = DST == 1 ? luma(r, g, b) : luma(r, g, b) | a << 8;
        o[(q * DST) >> 2] |= v << (8 * ((q * DST) & 3));
    }
}

// OutStrides in bytes: interleaved rows (pixel = DST * sizeof(T)) at any pitch, or planar (pixel = sizeof(T)); row 0: tight rows.
// All output addressing is 64-bit: one file's typed pixels may pass 4 GiB.
template <int SRC, int DST, bool PLANAR, typename T>
__global__ void __launch_bounds__(128) unfilter_typed_kernel(DecodeParams p, OutStrides os, PixelAffine pa)
{
    constexpr int ES = sizeof(T);
    const uint32_t f = blockIdx.y;
    const DecodeState st = p.state[f];
    if (st.status) return;
    const FileDesc& fd = p.files[f];
    if (fd.chans != SRC) return;                                                // the same for the whole CTA
    const uint32_t w = fd.w, h = fd.h, pitch = fd.pitch;
    const uint32_t x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;            // first pixel of the thread's group
    if (x0 >= w) return;
    const uint32_t npx = min(4u, w - x0);
    const bool full = npx == 4;
    const uint8_t* delta = p.delta + fd.delta_base + (size_t)x0 * SRC;
    uint8_t* out = p.d_out + fd.out_base + (size_t)x0 * (PLANAR ? 1u : DST) * ES;
    const size_t out_pitch = os.row ? os.row : (size_t)w * DST * ES, cs = os.chan;
    uint32_t acc[SRC];
#pragma unroll
    for (int i = 0; i < SRC; i++) acc[i] = 0;
    const bool summing = !st.stored;
    constexpr int kRowsAhead = 8;
    for (uint32_t y0 = 0; y0 < h; y0 += kRowsAhead) {
        uint32_t dd[kRowsAhead][SRC];
        load_delta_rows<SRC>(delta, pitch, y0, h, full, npx, dd);
#pragma unroll
        for (int j = 0; j < kRowsAhead; j++) {
            const uint32_t y = y0 + j;
            if (y >= h) break;
            uint32_t o[DST];
            if constexpr (DST >= 3) unfilter_row<SRC, DST>(acc, dd[j], summing, o);
            else {
                uint32_t px[SRC];
                unfilter_row<SRC, SRC>(acc, dd[j], summing, px);
                luma_row<SRC, DST>(px, o);
            }
            uint8_t* orow = out + (size_t)y * out_pitch;
            if (PLANAR) {                                                       // 4 * sizeof(T) contiguous bytes per plane
#pragma unroll
                for (int c = 0; c < DST; c++) {
                    uint32_t e[4];
#pragma unroll
                    for (int q = 0; q < 4; q++) e[q] = typed_value<T>(o, q * DST + c, c, pa);
                    uint8_t* a = orow + c * cs;
                    if (full) store_elems<T>(a, e);
                    else for (uint32_t q = 0; q < npx; q++) store_elem(a + ES * q, e[q], ES);
                }
            } else if (std::is_same<T, uint16_t>::value && full) {             // v * 257 is v in both bytes: 2 * DST words
                uint32_t wd[2 * DST];
#pragma unroll
                for (int i = 0; i < DST; i++) { wd[2 * i] = __byte_perm(o[i], 0, 0x1100); wd[2 * i + 1] = __byte_perm(o[i], 0, 0x3322); }
                if (((uintptr_t)orow & 3u) == 0u) store_elems<float, 2 * DST>(orow, wd);   // whole words where the address allows
                else {                                                          // tight rows of odd w * DST: 2-byte aligned
#pragma unroll
                    for (int k = 0; k < 4 * DST; k++) store_elem(orow + 2 * k, wd[k >> 1] >> (16 * (k & 1)), 2);
                }
            } else {                                                            // 4 * DST * sizeof(T) contiguous bytes
                uint32_t e[4 * DST];
#pragma unroll
                for (int k = 0; k < 4 * DST; k++) e[k] = typed_value<T>(o, k, k % DST, pa);
                if (full) store_elems<T>(orow, e);
                else {
#pragma unroll
                    for (int k = 0; k < 4 * DST; k++) if ((uint32_t)k < npx * DST) store_elem(orow + ES * k, e[k], ES);
                }
            }
        }
    }
}

// The planar layout exists for the float types at DST 3 and 4 only (the native calls write tight interleaved rows).
template <int SRC, int DST, typename T>
static void launch_one(const DecodeParams& p, const OutStrides& os, const PixelAffine& pa, dim3 g, cudaStream_t s)
{
    if constexpr (DST >= 3 && !std::is_integral<T>::value) {
        if (os.pixel == sizeof(T)) { unfilter_typed_kernel<SRC, DST, true, T><<<g, 128, 0, s>>>(p, os, pa); return; }
    }
    unfilter_typed_kernel<SRC, DST, false, T><<<g, 128, 0, s>>>(p, os, pa);
}
template <int SRC, typename T>
static void launch_src(const DecodeParams& p, const OutStrides& os, const PixelAffine& pa, uint32_t dst, dim3 g, cudaStream_t s)
{
    if (dst == 1) launch_one<SRC, 1, T>(p, os, pa, g, s);
    else if (dst == 2) launch_one<SRC, 2, T>(p, os, pa, g, s);
    else if (dst == 3) launch_one<SRC, 3, T>(p, os, pa, g, s);
    else launch_one<SRC, 4, T>(p, os, pa, g, s);
}

// one instantiation per source channel count in the call, as for unfilter_kernel; DST is desired, or for a native call's desired 0
// the file's own channel count
void launch_unfilter_typed(const DecodeParams& p, const OutStrides& os, const TypedOut& t, uint32_t desired, dim3 g, cudaStream_t s)
{
    with_out_type(t.dtype, [&](auto v) {
        using T = decltype(v);
        if (!p.chans || p.chans == 3) launch_src<3, T>(p, os, t.aff, desired ? desired : 3u, g, s);
        if (!p.chans || p.chans == 4) launch_src<4, T>(p, os, t.aff, desired ? desired : 4u, g, s);
    });
}

}  // namespace fpngb
