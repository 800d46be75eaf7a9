// fpng_b200/csrc/decode_resize_kernels.cu -- the last kernel of fpngb_decode_packed_resized_device: per-file crop and bilinear
// resize of the ragged decode's uint8 pixels into one fixed-size batch (include/fpng_b200.h, "resized decode", for the rule).
//
// One CTA per (file, tile of 32 output rows x 32 output columns); a CTA loops over tiles when there are more than the grid holds.
// The tile's source rows are those the taps of its first and last output rows span.  They are filtered horizontally, 8 at a
// time (one per warp, one output column per lane), into shared memory; each thread then accumulates 4 output columns of one
// output row vertically in registers, over the rows of the step its own taps cover.  Weights are computed on the fly from the
// per-axis rule, so any tap count works, from 1 up to a whole 3840-pixel crop resized to one pixel; no weight table is kept.
// All output addressing is 64-bit, and stores are the widest the address allows (store_elems).
// Native calls (FPNGB_RESIZE_NATIVE): the ragged decode holds every file as uint16 values in the 16-bit domain (S = uint16_t), any
// DST from 1 to 4; the resampled r is stored as cvt.rni.sat.u16(r), round_u8(r / 257) or T((r / 257) * scale + bias).
//
// decode_nearest_kernel takes decode_resize_kernel's place for FPNGB_RESIZE_NEAREST / FPNGB_RESIZE_NEAREST_EXACT.  It is a pure
// gather: each thread owns 4 consecutive output pixels of one row (the store group of the bilinear kernel), computes their source
// row and columns from the per-axis rule on the fly, and stores the source element converted to the ragged decode's element of the
// same call.  Threads of a warp own neighbouring groups of a row, so the stores are coalesced; the kernel is bound by them.
#include "decode.cuh"
#include "typed_store.cuh"
#include "../../include/fpng_b200.h"
#include <type_traits>

namespace fpngb {

constexpr uint32_t kRsThreads = 256;
constexpr uint32_t kRsCols = 32;            // output columns per tile: one per lane of the horizontal pass
constexpr uint32_t kRsRows = 32;            // output rows per tile: 32 rows x 8 groups of 4 columns in the vertical pass
constexpr uint32_t kRsStep = kRsThreads / 32;   // source rows filtered per step: one per warp

// Taps of output index i along one axis: source indices lo .. lo + size - 1 of a crop of length in; scale = in / out.  Every
// operation is a separately rounded fp32 one, as written in the header (no contraction into an FMA).
struct Span { int lo, size; float center, inv, norm; };

__device__ __forceinline__ float tap_weight(int j, float center, float inv)
{
    const float t = __fmul_rn(__fadd_rn(__fsub_rn((float)j, center), 0.5f), inv);
    return fmaxf(0.f, __fsub_rn(1.f, fabsf(t)));
}

__device__ __forceinline__ void span_bounds(int in, float scale, bool aa, uint32_t i, int& lo, int& hi, float& center)
{
    const float support = aa ? scale : 1.f;
    center = __fmul_rn(scale, __fadd_rn((float)i, 0.5f));
    lo = max((int)__fadd_rn(__fsub_rn(center, support), 0.5f), 0);           // truncation toward 0, as torch
    hi = min((int)__fadd_rn(__fadd_rn(center, support), 0.5f), in);
}

__device__ __forceinline__ Span axis_span(int in, float scale, bool aa, uint32_t i)
{
    int lo, hi;
    Span sp;
    span_bounds(in, scale, aa, i, lo, hi, sp.center);
    sp.lo = lo; sp.size = hi - lo; sp.inv = aa ? __fdiv_rn(1.f, scale) : 1.f;
    float sum = 0.f;
    for (int j = lo; j < hi; j++) sum = __fadd_rn(sum, tap_weight(j, sp.center, sp.inv));
    sp.norm = sum != 0.f ? __fdiv_rn(1.f, sum) : 1.f;
    return sp;
}

template <int DST>
__device__ __forceinline__ void load_px(const uint8_t* a, float (&v)[DST])
{
    if constexpr (DST == 4) {                                                   // 4-byte aligned: 16-byte file bases, 4-byte pixels
        const uint32_t u = __ldg(reinterpret_cast<const unsigned int*>(a));
#pragma unroll
        for (int c = 0; c < 4; c++) v[c] = (float)((u >> (8 * c)) & 0xFFu);
    } else {
#pragma unroll
        for (int c = 0; c < DST; c++) v[c] = (float)__ldg(a + c);
    }
}

// uint16 pixels of a native call: 8-byte (DST 4) or 4-byte (DST 2) aligned loads where the pixel size allows
template <int DST>
__device__ __forceinline__ void load_px16(const uint8_t* a, float (&v)[DST])
{
    if constexpr (DST == 4) {                                                   // 16-byte file bases, 8-byte pixels
        const uint2 u = __ldg(reinterpret_cast<const uint2*>(a));
        v[0] = (float)(u.x & 0xFFFFu); v[1] = (float)(u.x >> 16); v[2] = (float)(u.y & 0xFFFFu); v[3] = (float)(u.y >> 16);
    } else if constexpr (DST == 2) {
        const uint32_t u = __ldg(reinterpret_cast<const unsigned int*>(a));
        v[0] = (float)(u & 0xFFFFu); v[1] = (float)(u >> 16);
    } else {
#pragma unroll
        for (int c = 0; c < DST; c++) v[c] = (float)__ldg(reinterpret_cast<const unsigned short*>(a) + c);
    }
}

// the stored bits of the resampled value v of channel c: round_u8(v) for uint8, else T(v * scale[c] + bias[c]); from a uint16
// source (native calls): cvt.rni.sat.u16(v) for uint16, else the same rules applied to v / 257
template <typename T, typename S>
__device__ __forceinline__ uint32_t resized_bits(float v, int c, const PixelAffine& pa)
{
    if constexpr (std::is_same<T, uint16_t>::value) return typed_bits<T>(v);
    else {
        if constexpr (sizeof(S) == 2) v = __fdiv_rn(v, 257.0f);
        if constexpr (sizeof(T) == 1) return typed_bits<T>(v);
        else return typed_bits<T>(__fadd_rn(__fmul_rn(v, pa.scale[c]), pa.bias[c]));
    }
}

template <int DST, bool PLANAR, typename T, typename S = uint8_t>
__global__ void __launch_bounds__(kRsThreads) decode_resize_kernel(ResizeParams p, PixelAffine pa)
{
    constexpr int ES = sizeof(T), SS = sizeof(S);
    __shared__ float hbuf[kRsStep][kRsCols][DST];
    const uint32_t f = blockIdx.y;
    if (p.d_status[f] != 0) return;                                             // the same for the whole CTA
    const FileDesc& fd = p.files[f];
    const uint32_t w = fd.w;
    int top = 0, left = 0, bh = (int)fd.h, bw = (int)w;
    if (p.boxes) { const int32_t* b = p.boxes + (size_t)f * 4; top = b[0]; left = b[1]; bh = b[2]; bw = b[3]; }
    const uint8_t* src = p.px + p.px_offsets[f];
    const size_t pitch = (size_t)w * DST * SS;
    const float sx = __fdiv_rn((float)bw, (float)p.out_w), sy = __fdiv_rn((float)bh, (float)p.out_h);
    const bool aax = p.antialias && sx >= 1.f, aay = p.antialias && sy >= 1.f;
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, slot = threadIdx.x >> 3, grp = threadIdx.x & 7u;
    const uint32_t col_tiles = (p.out_w + kRsCols - 1) / kRsCols;
    const unsigned long long tiles = (unsigned long long)col_tiles * ((p.out_h + kRsRows - 1) / kRsRows);
    for (unsigned long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const uint32_t x0 = (uint32_t)(tile % col_tiles) * kRsCols, y0 = (uint32_t)(tile / col_tiles) * kRsRows;
        const uint32_t ox = x0 + lane, oy = y0 + slot;
        const Span hx = ox < p.out_w ? axis_span(bw, sx, aax, ox) : Span{0, 0, 0.f, 1.f, 0.f};
        const Span vy = oy < p.out_h ? axis_span(bh, sy, aay, oy) : Span{0, 0, 0.f, 1.f, 0.f};
        int r_lo, r_hi, unused_lo, unused_hi;
        float c0, c1;
        span_bounds(bh, sy, aay, y0, r_lo, unused_hi, c0);                                  // taps are monotone in the output index
        span_bounds(bh, sy, aay, min(y0 + kRsRows, p.out_h) - 1, unused_lo, r_hi, c1);
        float acc[4][DST];
#pragma unroll
        for (int q = 0; q < 4; q++)
#pragma unroll
            for (int c = 0; c < DST; c++) acc[q][c] = 0.f;
        for (int r0 = r_lo; r0 < r_hi; r0 += (int)kRsStep) {
            const int row = r0 + (int)warp;
            if (row < r_hi) {                                                   // horizontal pass: one source row per warp
                float h[DST];
#pragma unroll
                for (int c = 0; c < DST; c++) h[c] = 0.f;
                const uint8_t* s = src + (size_t)(top + row) * pitch + (size_t)(left + hx.lo) * DST * SS;
                for (int j = 0; j < hx.size; j++) {
                    const float wt = tap_weight(hx.lo + j, hx.center, hx.inv);
                    float v[DST];
                    if constexpr (SS == 2) load_px16<DST>(s + (size_t)j * DST * SS, v);
                    else load_px<DST>(s + (size_t)j * DST, v);
#pragma unroll
                    for (int c = 0; c < DST; c++) h[c] = fmaf(wt, v[c], h[c]);
                }
#pragma unroll
                for (int c = 0; c < DST; c++) hbuf[warp][lane][c] = __fmul_rn(h[c], hx.norm);
            }
            __syncthreads();
            const int r_end = min(r0 + (int)kRsStep, vy.lo + vy.size);         // vertical pass: the rows of the step this row's taps cover
            for (int r = max(r0, vy.lo); r < r_end; r++) {
                const float wt = tap_weight(r, vy.center, vy.inv);
#pragma unroll
                for (int q = 0; q < 4; q++)
#pragma unroll
                    for (int c = 0; c < DST; c++) acc[q][c] = fmaf(wt, hbuf[r - r0][4 * grp + q][c], acc[q][c]);
            }
            __syncthreads();
        }
        const uint32_t xg = x0 + 4 * grp;
        if (oy >= p.out_h || xg >= p.out_w) continue;
        const uint32_t npx = min(4u, p.out_w - xg);
        uint8_t* o = p.d_out + (size_t)f * p.image + (size_t)oy * p.row + (size_t)xg * p.pixel;
        if (PLANAR) {                                                           // 4 * sizeof(T) contiguous bytes per plane
#pragma unroll
            for (int c = 0; c < DST; c++) {
                uint32_t e[4];
#pragma unroll
                for (int q = 0; q < 4; q++) e[q] = resized_bits<T, S>(__fmul_rn(acc[q][c], vy.norm), c, pa);
                uint8_t* a = o + (size_t)c * p.chan;
                if (npx == 4) store_elems<T>(a, e);
                else for (uint32_t q = 0; q < npx; q++) store_elem(a + ES * q, e[q], ES);
            }
        } else {                                                                // 4 * DST * sizeof(T) contiguous bytes
            uint32_t e[4 * DST];
#pragma unroll
            for (int k = 0; k < 4 * DST; k++) e[k] = resized_bits<T, S>(__fmul_rn(acc[k / DST][k % DST], vy.norm), k % DST, pa);
            if (npx == 4) store_elems<T>(o, e);
            else {
#pragma unroll
                for (int k = 0; k < 4 * DST; k++) if ((uint32_t)k < npx * DST) store_elem(o + ES * k, e[k], ES);
            }
        }
    }
}

// source index of output index i along one axis of a crop of length in, scale = in / out: torch's nearest_neighbor_compute_source_index
// and nearest_neighbor_exact_compute_source_index (ATen/native/cuda/UpSample.cuh), each operation a separately rounded fp32 one
__device__ __forceinline__ int nearest_src(uint32_t i, float scale, int in, bool exact)
{
    const float x = exact ? __fadd_rn((float)i, 0.5f) : (float)i;
    return min((int)floorf(__fmul_rn(x, scale)), in - 1);
}

// DST elements of S at a (a pixel of the ragged decode's tight rows: 16-byte file bases, so aligned to DST * sizeof(S) where that is
// a power of two), as the widest load that alignment allows
template <int DST, typename S>
__device__ __forceinline__ void gather_px(const uint8_t* a, uint32_t (&v)[DST])
{
    constexpr int B = DST * (int)sizeof(S);
    if constexpr (B == 8) {
        const uint2 u = __ldg(reinterpret_cast<const uint2*>(a));
        v[0] = u.x & 0xFFFFu; v[1] = u.x >> 16; v[2] = u.y & 0xFFFFu; v[3] = u.y >> 16;
    } else if constexpr (B == 4 || B == 2) {
        const uint32_t u = B == 4 ? __ldg(reinterpret_cast<const unsigned int*>(a)) : __ldg(reinterpret_cast<const unsigned short*>(a));
        constexpr int SB = 8 * (int)sizeof(S);
#pragma unroll
        for (int c = 0; c < DST; c++) v[c] = (u >> (SB * c)) & ((1u << SB) - 1u);
    } else {
#pragma unroll
        for (int c = 0; c < DST; c++) v[c] = sizeof(S) == 2 ? __ldg(reinterpret_cast<const unsigned short*>(a) + c) : __ldg(a + c);
    }
}

// the stored bits of source element u of channel c: the element the ragged decode of the same call stores.  From a uint16 source
// (native calls: the 16-bit domain; index calls into uint16: the raw sample) u for uint16, u >> 8 for uint8, T(__fdiv_rn(u, 257) *
// scale + bias) for the float types; from a uint8 source u for uint8, T(u * scale + bias) for the float types.
template <typename T, typename S>
__device__ __forceinline__ uint32_t nearest_bits(uint32_t u, int c, const PixelAffine& pa)
{
    if constexpr (std::is_same<T, S>::value) return u;
    else if constexpr (std::is_same<T, uint8_t>::value) return u >> 8;
    else {
        const float x = sizeof(S) == 2 ? __fdiv_rn(__uint2float_rn(u), 257.0f) : __uint2float_rn(u);
        return typed_bits<T>(__fadd_rn(__fmul_rn(x, pa.scale[c]), pa.bias[c]));
    }
}

template <int DST, bool PLANAR, typename T, typename S>
__global__ void __launch_bounds__(kRsThreads) decode_nearest_kernel(ResizeParams p, PixelAffine pa)
{
    constexpr int ES = sizeof(T), SS = sizeof(S);
    const uint32_t f = blockIdx.y;
    if (p.d_status[f] != 0) return;                                             // the same for the whole CTA
    const FileDesc& fd = p.files[f];
    int top = 0, left = 0, bh = (int)fd.h, bw = (int)fd.w;
    if (p.boxes) { const int32_t* b = p.boxes + (size_t)f * 4; top = b[0]; left = b[1]; bh = b[2]; bw = b[3]; }
    const uint8_t* src = p.px + p.px_offsets[f] + ((size_t)top * fd.w + left) * DST * SS;
    const size_t pitch = (size_t)fd.w * DST * SS;
    const float sx = __fdiv_rn((float)bw, (float)p.out_w), sy = __fdiv_rn((float)bh, (float)p.out_h);
    const bool exact = p.nearest == 2;
    // groups of 4 output pixels: gx per row; each thread steps through them by the grid's thread count, carried as (row, group)
    const uint32_t gx = (p.out_w + 3) / 4;
    const unsigned long long groups = (unsigned long long)gx * p.out_h, step = (unsigned long long)gridDim.x * blockDim.x;
    const unsigned long long g0 = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g0 >= groups) return;
    uint32_t oy = (uint32_t)(g0 / gx), xq = (uint32_t)(g0 % gx);
    const uint32_t dy = (uint32_t)(step / gx), dq = (uint32_t)(step % gx);
    for (unsigned long long g = g0; g < groups; g += step) {
        const uint32_t xg = 4 * xq, npx = min(4u, p.out_w - xg);
        const uint8_t* srow = src + (size_t)nearest_src(oy, sy, bh, exact) * pitch;
        uint32_t v[4][DST];
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const int x = (uint32_t)q < npx ? nearest_src(xg + q, sx, bw, exact) : 0;
            gather_px<DST, S>(srow + (size_t)x * DST * SS, v[q]);
        }
        uint8_t* o = p.d_out + (size_t)f * p.image + (size_t)oy * p.row + (size_t)xg * p.pixel;
        if (PLANAR) {                                                           // 4 * sizeof(T) contiguous bytes per plane
#pragma unroll
            for (int c = 0; c < DST; c++) {
                uint32_t e[4];
#pragma unroll
                for (int q = 0; q < 4; q++) e[q] = nearest_bits<T, S>(v[q][c], c, pa);
                uint8_t* a = o + (size_t)c * p.chan;
                if (npx == 4) store_elems<T>(a, e);
                else for (uint32_t q = 0; q < npx; q++) store_elem(a + ES * q, e[q], ES);
            }
        } else {                                                                // 4 * DST * sizeof(T) contiguous bytes
            uint32_t e[4 * DST];
#pragma unroll
            for (int k = 0; k < 4 * DST; k++) e[k] = nearest_bits<T, S>(v[k / DST][k % DST], k % DST, pa);
            if (npx == 4) store_elems<T>(o, e);
            else {
#pragma unroll
                for (int k = 0; k < 4 * DST; k++) if ((uint32_t)k < npx * DST) store_elem(o + ES * k, e[k], ES);
            }
        }
        oy += dy; xq += dq;
        if (xq >= gx) { xq -= gx; oy++; }
    }
}

template <int DST, typename T, typename S>
static void launch_nearest_dst(const ResizeParams& p, const PixelAffine& pa, uint32_t n, cudaStream_t s)
{
    const unsigned long long groups = (unsigned long long)((p.out_w + 3) / 4) * p.out_h, ctas = (groups + kRsThreads - 1) / kRsThreads;
    const dim3 g((uint32_t)(ctas < 65535ull ? ctas : 65535ull), n);
    if constexpr (DST > 1) {                            // one channel: planar and interleaved address the same elements
        if (p.pixel == sizeof(T)) { decode_nearest_kernel<DST, true, T, S><<<g, kRsThreads, 0, s>>>(p, pa); return; }
    }
    decode_nearest_kernel<DST, false, T, S><<<g, kRsThreads, 0, s>>>(p, pa);
}

// the nearest resize: S uint16 for native calls and uint16 index calls (DST 1 .. 4), else uint8 (DST 3 / 4, or 1 for a uint8 index call)
static void launch_decode_nearest(const ResizeParams& p, const TypedOut& t, uint32_t src_dtype, uint32_t n, uint32_t desired, cudaStream_t s)
{
    with_out_type(t.dtype, [&](auto v) {
        using T = decltype(v);
        if (src_dtype == FPNGB_DTYPE_UINT16) {
            if (desired == 1) launch_nearest_dst<1, T, uint16_t>(p, t.aff, n, s);
            else if (desired == 2) launch_nearest_dst<2, T, uint16_t>(p, t.aff, n, s);
            else if (desired == 3) launch_nearest_dst<3, T, uint16_t>(p, t.aff, n, s);
            else launch_nearest_dst<4, T, uint16_t>(p, t.aff, n, s);
        } else if constexpr (!std::is_same<T, uint16_t>::value) {
            if (desired == 1) { if constexpr (std::is_same<T, uint8_t>::value) launch_nearest_dst<1, T, uint8_t>(p, t.aff, n, s); }
            else if (desired == 3) launch_nearest_dst<3, T, uint8_t>(p, t.aff, n, s);
            else launch_nearest_dst<4, T, uint8_t>(p, t.aff, n, s);
        }
    });
}

template <int DST, typename T, typename S>
static void launch_dst(const ResizeParams& p, const PixelAffine& pa, dim3 g, cudaStream_t s)
{
    if constexpr (DST > 1) {                            // one channel: planar and interleaved address the same elements
        if (p.pixel == sizeof(T)) { decode_resize_kernel<DST, true, T, S><<<g, kRsThreads, 0, s>>>(p, pa); return; }
    }
    decode_resize_kernel<DST, false, T, S><<<g, kRsThreads, 0, s>>>(p, pa);
}

// src_dtype: the ragged decode's output, FPNGB_DTYPE_UINT16 for a native call (DST 1 .. 4), else 0 (uint8, DST 3 or 4)
void launch_decode_resize(const ResizeParams& p, const TypedOut& t, uint32_t src_dtype, uint32_t n, uint32_t desired, cudaStream_t s)
{
    if (p.nearest) { launch_decode_nearest(p, t, src_dtype, n, desired, s); return; }
    const unsigned long long tiles = (unsigned long long)((p.out_w + kRsCols - 1) / kRsCols) * ((p.out_h + kRsRows - 1) / kRsRows);
    const dim3 g((uint32_t)(tiles < 65535ull ? tiles : 65535ull), n);
    with_out_type(t.dtype, [&](auto v) {
        using T = decltype(v);
        if (src_dtype == FPNGB_DTYPE_UINT16) {
            if (desired == 1) launch_dst<1, T, uint16_t>(p, t.aff, g, s);
            else if (desired == 2) launch_dst<2, T, uint16_t>(p, t.aff, g, s);
            else if (desired == 3) launch_dst<3, T, uint16_t>(p, t.aff, g, s);
            else launch_dst<4, T, uint16_t>(p, t.aff, g, s);
        } else if constexpr (!std::is_same<T, uint16_t>::value) {
            if (desired == 3) launch_dst<3, T, uint8_t>(p, t.aff, g, s);
            else launch_dst<4, T, uint8_t>(p, t.aff, g, s);
        }
    });
}

}  // namespace fpngb
