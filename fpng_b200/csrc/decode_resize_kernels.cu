// fpng_b200/csrc/decode_resize_kernels.cu -- the last kernel of fpngb_decode_packed_resized_device: per-file crop and bilinear
// resize of the ragged decode's uint8 pixels into one fixed-size batch (include/fpng_b200.h, "resized decode", for the rule).
//
// One CTA per (file, tile of 32 output rows x 32 output columns); a CTA loops over tiles when there are more than the grid holds.
// The tile's source rows are those the taps of its first and last output rows span.  They are filtered horizontally, 8 at a
// time (one per warp, one output column per lane), into shared memory; each thread then accumulates 4 output columns of one
// output row vertically in registers, over the rows of the step its own taps cover.  Weights are computed on the fly from the
// per-axis rule, so any tap count works, from 1 up to a whole 3840-pixel crop resized to one pixel; no weight table is kept.
// All output addressing is 64-bit, and stores are the widest the address allows (store_elems).
// Views (fpngb_decode_packed_views_device): CTA row blockIdx.y is one output image, a view of a file: its box resized to its own
// rh x rw, flipped, and placed at an offset on the canvas, fill elsewhere (view_geom).  The flip maps an output index to the resized
// index before any tap is computed, so each resized value is computed exactly as in the resized call; without a view table the
// geometry is that call's (box, resize to the canvas, offset 0, no flips), so both calls run the same code.
// Native calls (FPNGB_RESIZE_NATIVE): the ragged decode holds every file as uint16 values in the 16-bit domain (S = uint16_t), any
// DST from 1 to 4; the resampled r is stored as cvt.rni.sat.u16(r), round_u8(r / 257) or T((r / 257) * scale + bias).
//
// Bicubic (FPNGB_RESIZE_BICUBIC, the CUBIC instantiations): the same tiles and passes with torch's bicubic taps and weights.  The
// antialiased filter keeps the span rule with support 2 * max(scale, 1); the plain filter has 4 taps at floorf(real) - 1 .. + 2
// that may lie outside the crop: the staged rows and the column loads read the clamped index, so the border of the crop (not of
// the file) is replicated, and the staged row range, taken from the unclamped taps, runs up to 2 rows past either end of the crop.
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

// torch's cubic convolution kernel at distance d >= 0 (A = -0.75 plain, a = -0.5 antialiased), each operation separately rounded
__device__ __forceinline__ float cubic_weight(float d, float a)
{
    if (d < 1.f) return __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(a, 2.f), d), __fadd_rn(a, 3.f)), d), d), 1.f);
    if (d < 2.f) return __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(a, d), __fmul_rn(5.f, a)), d), __fmul_rn(8.f, a)), d),
                                  __fmul_rn(4.f, a));
    return 0.f;
}

// Bicubic taps of output index i (the CUBIC counterparts of span_bounds, tap_weight and axis_span).  Antialiased: the span rule
// with support 2 * scale (2 below scale 1) and invscale 1 / scale (1 below scale 1), at every scale.  Plain: real = scale * (i +
// 0.5) - 0.5, unclamped; lo = floorf(real) - 1, 4 taps; center holds t = real - floorf(real); the indices are clamped by the loads.
__device__ __forceinline__ void cubic_bounds(int in, float scale, bool aa, uint32_t i, int& lo, int& hi, float& center)
{
    if (aa) {
        const float support = scale >= 1.f ? __fmul_rn(2.f, scale) : 2.f;
        center = __fmul_rn(scale, __fadd_rn((float)i, 0.5f));
        lo = max((int)__fadd_rn(__fsub_rn(center, support), 0.5f), 0);
        hi = min((int)__fadd_rn(__fadd_rn(center, support), 0.5f), in);
    } else {
        const float real = __fsub_rn(__fmul_rn(scale, __fadd_rn((float)i, 0.5f)), 0.5f), x0 = floorf(real);
        center = __fsub_rn(real, x0);
        lo = (int)x0 - 1; hi = lo + 4;
    }
}

// weight of tap j: plain taps k = j - lo at distances t + 1, t, 1 - t, 2 - t (not normalised)
__device__ __forceinline__ float cubic_tap(int j, const Span& sp, bool aa)
{
    if (aa) return cubic_weight(fabsf(__fmul_rn(__fadd_rn(__fsub_rn((float)j, sp.center), 0.5f), sp.inv)), -0.5f);
    const int k = j - sp.lo;
    const float t = sp.center;
    const float d = k == 0 ? __fadd_rn(t, 1.f) : k == 1 ? t : k == 2 ? __fsub_rn(1.f, t) : __fsub_rn(2.f, t);
    return cubic_weight(d, -0.75f);
}

__device__ __forceinline__ Span cubic_span(int in, float scale, bool aa, uint32_t i)
{
    int lo, hi;
    Span sp;
    cubic_bounds(in, scale, aa, i, lo, hi, sp.center);
    sp.lo = lo; sp.size = hi - lo; sp.inv = aa && scale >= 1.f ? __fdiv_rn(1.f, scale) : 1.f; sp.norm = 1.f;
    if (aa) {
        float sum = 0.f;
        for (int j = lo; j < hi; j++) sum = __fadd_rn(sum, cubic_tap(j, sp, true));
        sp.norm = sum != 0.f ? __fdiv_rn(1.f, sum) : 1.f;
    }
    return sp;
}

template <bool CUBIC>
__device__ __forceinline__ void filter_bounds(int in, float scale, bool aa, uint32_t i, int& lo, int& hi, float& center)
{
    if constexpr (CUBIC) cubic_bounds(in, scale, aa, i, lo, hi, center);
    else span_bounds(in, scale, aa, i, lo, hi, center);
}

template <bool CUBIC>
__device__ __forceinline__ Span filter_span(int in, float scale, bool aa, uint32_t i)
{
    if constexpr (CUBIC) return cubic_span(in, scale, aa, i);
    else return axis_span(in, scale, aa, i);
}

template <bool CUBIC>
__device__ __forceinline__ float filter_tap(int j, const Span& sp, bool aa)
{
    if constexpr (CUBIC) return cubic_tap(j, sp, aa);
    else return tap_weight(j, sp.center, sp.inv);
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

// The geometry of output image blockIdx.y.  With a view table: row blockIdx.y, and its status (include/fpng_b200.h, "views"),
// written by the CTA with blockIdx.x == 0; without one: file blockIdx.y, its box or whole image resized to the canvas at offset 0.
// The placed image covers canvas rows [y_in0, y_in1) and columns [x_in0, x_in1) (empty when it lies off the canvas).
struct ViewGeom {
    uint32_t f; int status;
    int top, left, bh, bw;                  // the crop box
    int rh, rw, oy, ox;                     // resized size and offset on the canvas
    bool hflip, vflip;
    int y_in0, y_in1, x_in0, x_in1;
};

__device__ __forceinline__ ViewGeom view_geom(const ResizeParams& p)
{
    ViewGeom g;
    const uint32_t v = blockIdx.y;
    g.top = 0; g.left = 0; g.rh = (int)p.out_h; g.rw = (int)p.out_w; g.oy = 0; g.ox = 0; g.hflip = g.vflip = false;
    if (!p.views) {
        g.f = v;
        g.status = p.d_status[v];
        if (p.boxes) { const int32_t* b = p.boxes + (size_t)v * 4; g.top = b[0]; g.left = b[1]; g.bh = b[2]; g.bw = b[3]; }
        else { g.bh = (int)p.files[v].h; g.bw = (int)p.files[v].w; }
    } else {
        const int32_t* r = p.views + (size_t)v * 10;
        const int file = r[0];
        g.f = 0; g.top = r[1]; g.left = r[2]; g.bh = r[3]; g.bw = r[4]; g.rh = r[5]; g.rw = r[6]; g.oy = r[7]; g.ox = r[8];
        const uint32_t flags = (uint32_t)r[9];
        constexpr int kLim = 1 << 24;
        if (file < 0 || (uint32_t)file >= p.n) g.status = FPNGB_DECODE_BAD_VIEW;
        else if ((g.status = p.d_status[file]) != 0) {}
        else if (g.bh < 1 || g.bw < 1 || g.top < 0 || g.left < 0 || (long long)g.top + g.bh > p.files[file].h ||
                 (long long)g.left + g.bw > p.files[file].w)
            g.status = FPNGB_DECODE_BAD_CROP;
        else if (g.rh < 1 || g.rh > kLim || g.rw < 1 || g.rw > kLim || g.oy < -kLim || g.oy > kLim || g.ox < -kLim || g.ox > kLim ||
                 (flags & ~(uint32_t)(FPNGB_VIEW_HFLIP | FPNGB_VIEW_VFLIP)))
            g.status = FPNGB_DECODE_BAD_VIEW;
        if (blockIdx.x == 0 && threadIdx.x == 0) p.view_status[v] = g.status;
        if (g.status == 0) g.f = (uint32_t)file;
        g.hflip = flags & FPNGB_VIEW_HFLIP; g.vflip = flags & FPNGB_VIEW_VFLIP;
    }
    g.y_in0 = max(g.oy, 0); g.y_in1 = min(g.oy + g.rh, (int)p.out_h);
    g.x_in0 = max(g.ox, 0); g.x_in1 = min(g.ox + g.rw, (int)p.out_w);
    return g;
}

// resized index of canvas index o (inside the placed image) along an axis placed at offset at, of resized length len
__device__ __forceinline__ uint32_t resized_index(int o, int at, int len, bool flip) { return (uint32_t)(flip ? len - 1 - (o - at) : o - at); }

template <int DST, bool PLANAR, typename T, typename S = uint8_t, bool CUBIC = false>
__global__ void __launch_bounds__(kRsThreads) decode_resize_kernel(ResizeParams p, PixelAffine pa)
{
    constexpr int ES = sizeof(T), SS = sizeof(S);
    __shared__ float hbuf[kRsStep][kRsCols][DST];
    const ViewGeom g = view_geom(p);
    if (g.status != 0) return;                                                  // the same for the whole CTA
    const int top = g.top, left = g.left, bh = g.bh, bw = g.bw;
    const uint8_t* src = p.px + p.px_offsets[g.f];
    const size_t pitch = (size_t)p.files[g.f].w * DST * SS;
    const float sx = __fdiv_rn((float)bw, (float)g.rw), sy = __fdiv_rn((float)bh, (float)g.rh);
    // bilinear: the antialiased span equals the plain one below scale 1; bicubic: the antialiased filter applies at every scale
    const bool aax = p.antialias && (CUBIC || sx >= 1.f), aay = p.antialias && (CUBIC || sy >= 1.f);
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, slot = threadIdx.x >> 3, grp = threadIdx.x & 7u;
    const uint32_t col_tiles = (p.out_w + kRsCols - 1) / kRsCols;
    const unsigned long long tiles = (unsigned long long)col_tiles * ((p.out_h + kRsRows - 1) / kRsRows);
    for (unsigned long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const uint32_t x0 = (uint32_t)(tile % col_tiles) * kRsCols, y0 = (uint32_t)(tile / col_tiles) * kRsRows;
        const uint32_t ox = x0 + lane, oy = y0 + slot;
        const bool row_in = (int)oy >= g.y_in0 && (int)oy < g.y_in1;
        const Span hx = (int)ox >= g.x_in0 && (int)ox < g.x_in1 ? filter_span<CUBIC>(bw, sx, aax, resized_index((int)ox, g.ox, g.rw, g.hflip))
                                                               : Span{0, 0, 0.f, 1.f, 0.f};
        const Span vy = row_in ? filter_span<CUBIC>(bh, sy, aay, resized_index((int)oy, g.oy, g.rh, g.vflip)) : Span{0, 0, 0.f, 1.f, 0.f};
        // source rows: the taps of the tile's first and last in-image output rows (taps are monotone in the resized index, which
        // runs backwards under VFLIP); none when no pixel of the tile lies in the placed image
        int r_lo = 0, r_hi = 0, unused_lo, unused_hi;
        const int ya = max((int)y0, g.y_in0), yb = min((int)y0 + (int)kRsRows, g.y_in1) - 1;
        if (ya <= yb && max((int)x0, g.x_in0) < min((int)x0 + (int)kRsCols, g.x_in1)) {
            const uint32_t ia = resized_index(g.vflip ? yb : ya, g.oy, g.rh, g.vflip), ib = resized_index(g.vflip ? ya : yb, g.oy, g.rh, g.vflip);
            float c0, c1;
            filter_bounds<CUBIC>(bh, sy, aay, ia, r_lo, unused_hi, c0);
            filter_bounds<CUBIC>(bh, sy, aay, ib, unused_lo, r_hi, c1);
        }
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
                if constexpr (CUBIC) {                                          // plain taps past the crop read its edge
                    const uint8_t* s = src + (size_t)(top + min(max(row, 0), bh - 1)) * pitch + (size_t)left * DST * SS;
                    for (int j = hx.lo; j < hx.lo + hx.size; j++) {
                        const float wt = cubic_tap(j, hx, aax);
                        const size_t at = (size_t)min(max(j, 0), bw - 1) * DST * SS;
                        float v[DST];
                        if constexpr (SS == 2) load_px16<DST>(s + at, v);
                        else load_px<DST>(s + at, v);
#pragma unroll
                        for (int c = 0; c < DST; c++) h[c] = fmaf(wt, v[c], h[c]);
                    }
                } else {
                    const uint8_t* s = src + (size_t)(top + row) * pitch + (size_t)(left + hx.lo) * DST * SS;
                    for (int j = 0; j < hx.size; j++) {
                        const float wt = tap_weight(hx.lo + j, hx.center, hx.inv);
                        float v[DST];
                        if constexpr (SS == 2) load_px16<DST>(s + (size_t)j * DST * SS, v);
                        else load_px<DST>(s + (size_t)j * DST, v);
#pragma unroll
                        for (int c = 0; c < DST; c++) h[c] = fmaf(wt, v[c], h[c]);
                    }
                }
#pragma unroll
                for (int c = 0; c < DST; c++) hbuf[warp][lane][c] = __fmul_rn(h[c], hx.norm);
            }
            __syncthreads();
            const int r_end = min(r0 + (int)kRsStep, vy.lo + vy.size);         // vertical pass: the rows of the step this row's taps cover
            for (int r = max(r0, vy.lo); r < r_end; r++) {
                const float wt = filter_tap<CUBIC>(r, vy, aay);
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
        bool in[4];                                                             // else the fill, a source value of the call
#pragma unroll
        for (int q = 0; q < 4; q++) in[q] = row_in && (int)(xg + q) >= g.x_in0 && (int)(xg + q) < g.x_in1;
        uint8_t* o = p.d_out + (size_t)blockIdx.y * p.image + (size_t)oy * p.row + (size_t)xg * p.pixel;
        if (PLANAR) {                                                           // 4 * sizeof(T) contiguous bytes per plane
#pragma unroll
            for (int c = 0; c < DST; c++) {
                uint32_t e[4];
#pragma unroll
                for (int q = 0; q < 4; q++) e[q] = resized_bits<T, S>(in[q] ? __fmul_rn(acc[q][c], vy.norm) : (float)p.fill[c], c, pa);
                uint8_t* a = o + (size_t)c * p.chan;
                if (npx == 4) store_elems<T>(a, e);
                else for (uint32_t q = 0; q < npx; q++) store_elem(a + ES * q, e[q], ES);
            }
        } else {                                                                // 4 * DST * sizeof(T) contiguous bytes
            uint32_t e[4 * DST];
#pragma unroll
            for (int k = 0; k < 4 * DST; k++)
                e[k] = resized_bits<T, S>(in[k / DST] ? __fmul_rn(acc[k / DST][k % DST], vy.norm) : (float)p.fill[k % DST], k % DST, pa);
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
    const ViewGeom vg = view_geom(p);
    if (vg.status != 0) return;                                                  // the same for the whole CTA
    const uint32_t fw = p.files[vg.f].w;
    const int bh = vg.bh, bw = vg.bw;
    const uint8_t* src = p.px + p.px_offsets[vg.f] + ((size_t)vg.top * fw + vg.left) * DST * SS;
    const size_t pitch = (size_t)fw * DST * SS;
    const float sx = __fdiv_rn((float)bw, (float)vg.rw), sy = __fdiv_rn((float)bh, (float)vg.rh);
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
        const bool row_in = (int)oy >= vg.y_in0 && (int)oy < vg.y_in1;
        const uint8_t* srow = src + (row_in ? (size_t)nearest_src(resized_index((int)oy, vg.oy, vg.rh, vg.vflip), sy, bh, exact) * pitch : 0);
        uint32_t v[4][DST];
#pragma unroll
        for (int q = 0; q < 4; q++) {
            if (row_in && (uint32_t)q < npx && (int)(xg + q) >= vg.x_in0 && (int)(xg + q) < vg.x_in1) {
                const int x = nearest_src(resized_index((int)(xg + q), vg.ox, vg.rw, vg.hflip), sx, bw, exact);
                gather_px<DST, S>(srow + (size_t)x * DST * SS, v[q]);
            } else {                                                            // the fill, a source value of the call
#pragma unroll
                for (int c = 0; c < DST; c++) v[q][c] = p.fill[c];
            }
        }
        uint8_t* o = p.d_out + (size_t)blockIdx.y * p.image + (size_t)oy * p.row + (size_t)xg * p.pixel;
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
static void launch_nearest_dst(const ResizeParams& p, const PixelAffine& pa, uint32_t m, cudaStream_t s)
{
    const unsigned long long groups = (unsigned long long)((p.out_w + 3) / 4) * p.out_h, ctas = (groups + kRsThreads - 1) / kRsThreads;
    const dim3 g((uint32_t)(ctas < 65535ull ? ctas : 65535ull), m);
    if constexpr (DST > 1) {                            // one channel: planar and interleaved address the same elements
        if (p.pixel == sizeof(T)) { decode_nearest_kernel<DST, true, T, S><<<g, kRsThreads, 0, s>>>(p, pa); return; }
    }
    decode_nearest_kernel<DST, false, T, S><<<g, kRsThreads, 0, s>>>(p, pa);
}

// the nearest resize (m: output images, the grid's y): S uint16 for native calls and uint16 index calls (DST 1 .. 4), else uint8 (DST 3 / 4, or 1 for a uint8 index call)
static void launch_decode_nearest(const ResizeParams& p, const TypedOut& t, uint32_t src_dtype, uint32_t m, uint32_t desired, cudaStream_t s)
{
    with_out_type(t.dtype, [&](auto v) {
        using T = decltype(v);
        if (src_dtype == FPNGB_DTYPE_UINT16) {
            if (desired == 1) launch_nearest_dst<1, T, uint16_t>(p, t.aff, m, s);
            else if (desired == 2) launch_nearest_dst<2, T, uint16_t>(p, t.aff, m, s);
            else if (desired == 3) launch_nearest_dst<3, T, uint16_t>(p, t.aff, m, s);
            else launch_nearest_dst<4, T, uint16_t>(p, t.aff, m, s);
        } else if constexpr (!std::is_same<T, uint16_t>::value) {
            if (desired == 1) { if constexpr (std::is_same<T, uint8_t>::value) launch_nearest_dst<1, T, uint8_t>(p, t.aff, m, s); }
            else if (desired == 3) launch_nearest_dst<3, T, uint8_t>(p, t.aff, m, s);
            else launch_nearest_dst<4, T, uint8_t>(p, t.aff, m, s);
        }
    });
}

template <int DST, typename T, typename S, bool CUBIC>
static void launch_filter(const ResizeParams& p, const PixelAffine& pa, dim3 g, cudaStream_t s)
{
    if constexpr (DST > 1) {                            // one channel: planar and interleaved address the same elements
        if (p.pixel == sizeof(T)) { decode_resize_kernel<DST, true, T, S, CUBIC><<<g, kRsThreads, 0, s>>>(p, pa); return; }
    }
    decode_resize_kernel<DST, false, T, S, CUBIC><<<g, kRsThreads, 0, s>>>(p, pa);
}

template <int DST, typename T, typename S>
static void launch_dst(const ResizeParams& p, const PixelAffine& pa, bool cubic, dim3 g, cudaStream_t s)
{
    if (cubic) launch_filter<DST, T, S, true>(p, pa, g, s);
    else launch_filter<DST, T, S, false>(p, pa, g, s);
}

// src_dtype: the ragged decode's output, FPNGB_DTYPE_UINT16 for a native call (DST 1 .. 4), else 0 (uint8, DST 3 or 4); m: output
// images (files, or views with p.views); cubic: FPNGB_RESIZE_BICUBIC (the bilinear kernel's other filter)
void launch_decode_resize(const ResizeParams& p, const TypedOut& t, uint32_t src_dtype, uint32_t m, uint32_t desired, bool cubic,
                          cudaStream_t s)
{
    if (p.nearest) { launch_decode_nearest(p, t, src_dtype, m, desired, s); return; }
    const unsigned long long tiles = (unsigned long long)((p.out_w + kRsCols - 1) / kRsCols) * ((p.out_h + kRsRows - 1) / kRsRows);
    const dim3 g((uint32_t)(tiles < 65535ull ? tiles : 65535ull), m);
    with_out_type(t.dtype, [&](auto v) {
        using T = decltype(v);
        if (src_dtype == FPNGB_DTYPE_UINT16) {
            if (desired == 1) launch_dst<1, T, uint16_t>(p, t.aff, cubic, g, s);
            else if (desired == 2) launch_dst<2, T, uint16_t>(p, t.aff, cubic, g, s);
            else if (desired == 3) launch_dst<3, T, uint16_t>(p, t.aff, cubic, g, s);
            else launch_dst<4, T, uint16_t>(p, t.aff, cubic, g, s);
        } else if constexpr (!std::is_same<T, uint16_t>::value) {
            if (desired == 3) launch_dst<3, T, uint8_t>(p, t.aff, cubic, g, s);
            else launch_dst<4, T, uint8_t>(p, t.aff, cubic, g, s);
        }
    });
}

}  // namespace fpngb
