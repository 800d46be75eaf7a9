// fpng_b200/csrc/layout.h -- the pixel formats and layouts of the device entry points (include/fpng_b200.h, "Pixel layouts").
// A batch is an [n, h, w, chans] array of elements: element (i, y, x, c) at byte base + i*image + y*row + x*pixel + c*chan.
// Depends on the C headers only, so that the argument rules can be compiled and tested without CUDA.
#pragma once
#include "../../include/fpng_b200.h"
#include <math.h>
#include <stddef.h>
#include <stdint.h>

namespace fpngb {

// The element format of a call: dtype 0 is uint8 (the calls without a fpngb_pixel_format), else an FPNGB_DTYPE_* value with the
// per-channel scale and bias of the channels in use (the others 0).
struct PixelFormat {
    uint32_t dtype;
    uint32_t elem;                      // bytes per element
    float scale[4], bias[4];
};

inline PixelFormat uint8_format() { return PixelFormat{0, 1, {0, 0, 0, 0}, {0, 0, 0, 0}}; }

// The format of a *_typed call whose largest channel count is chans: FPNGB_ERR_INVALID_ARG for a NULL fmt, a dtype other than the
// three float types, or a scale or bias entry in use (index < chans) that is not finite.
inline int parse_format(const fpngb_pixel_format* fmt, uint32_t chans, PixelFormat& f)
{
    if (!fmt || (fmt->dtype != FPNGB_DTYPE_FLOAT32 && fmt->dtype != FPNGB_DTYPE_FLOAT16 && fmt->dtype != FPNGB_DTYPE_BFLOAT16))
        return FPNGB_ERR_INVALID_ARG;
    f = PixelFormat{fmt->dtype, fmt->dtype == FPNGB_DTYPE_FLOAT32 ? 4u : 2u, {0, 0, 0, 0}, {0, 0, 0, 0}};
    for (uint32_t c = 0; c < chans && c < 4; c++) {
        if (!isfinite(fmt->scale[c]) || !isfinite(fmt->bias[c])) return FPNGB_ERR_INVALID_ARG;
        f.scale[c] = fmt->scale[c]; f.bias[c] = fmt->bias[c];
    }
    return FPNGB_OK;
}

struct Layout {
    uint64_t image, row, pixel, chan;   // byte strides after canonicalisation
    bool planar;                        // one plane per channel: pixel is one element; else interleaved: pixel is chans elements, chan one
};

// Canonicalises the strides of size-1 dimensions (they address nothing, so they get the values of a tightly packed batch:
// the 16-byte alignment tests of the staged loaders then see only strides that matter) and classifies the layout.
// False: neither interleaved nor planar.
inline bool classify_layout(uint64_t image, uint64_t row, uint64_t pixel, uint64_t chan, uint32_t n, uint32_t h, uint32_t w, uint32_t chans,
                            Layout& L)
{
    if (w == 1) pixel = chan == 1 ? chans : 1;
    const bool interleaved = pixel == chans && chan == 1;
    const bool planar = !interleaved && pixel == 1 && chan >= 1;
    if (!interleaved && !planar) return false;
    if (h == 1) row = interleaved ? (uint64_t)w * chans : w;
    if (n == 1) image = (uint64_t)h * row;
    L = Layout{image, row, pixel, chan, planar};
    return true;
}

// tight interleaved rows of w pixels of chans bytes, consecutive images image bytes apart
inline Layout tight_layout(uint32_t w, uint32_t chans, uint64_t image) { return Layout{image, (uint64_t)w * chans, chans, 1, false}; }

// Offset of the last byte, false on 64-bit overflow or when base + offset wraps the address space.
inline bool layout_span(const void* base, const Layout& L, uint32_t n, uint32_t h, uint32_t w, uint32_t chans, uint64_t& last)
{
    const uint64_t size[4] = {n, h, w, chans}, stride[4] = {L.image, L.row, L.pixel, L.chan};
    unsigned __int128 s = 0;
    for (int k = 0; k < 4; k++) s += (unsigned __int128)(size[k] - 1) * stride[k];
    if (s > (unsigned __int128)(UINT64_MAX - (uint64_t)(uintptr_t)base)) return false;
    last = (uint64_t)s;
    return true;
}

// No two (i, y, x, c) of an output layout share a byte: with the dimensions of size > 1 ordered by stride, every stride is
// at least the span of the dimensions below it plus one.
inline bool layout_disjoint(const Layout& L, uint32_t n, uint32_t h, uint32_t w, uint32_t chans)
{
    uint64_t size[4] = {n, h, w, chans}, stride[4] = {L.image, L.row, L.pixel, L.chan};
    int m = 0;
    uint64_t sz[4], st[4];
    for (int k = 0; k < 4; k++) if (size[k] > 1) { sz[m] = size[k]; st[m] = stride[k]; m++; }
    for (int a = 1; a < m; a++)                                     // insertion sort by stride
        for (int b = a; b > 0 && st[b] < st[b - 1]; b--) { uint64_t t = st[b]; st[b] = st[b - 1]; st[b - 1] = t; t = sz[b]; sz[b] = sz[b - 1]; sz[b - 1] = t; }
    unsigned __int128 span = 0;
    for (int k = 0; k < m; k++) {
        if ((unsigned __int128)st[k] < span + 1) return false;
        span += (unsigned __int128)st[k] * (sz[k] - 1);
    }
    return true;
}

// The byte layout L of an [n, h, w, chans] array of elem-byte elements at base, given its byte strides.  FPNGB_ERR_ALIGNMENT unless
// base and every stride are multiples of elem; FPNGB_ERR_INVALID_ARG unless the strides divided by elem form an interleaved or
// planar layout (classify_layout) whose last element lies inside the address space.  An output must also be disjoint: no two
// elements share a byte.  An input's strides must stay inside 64 bits when scaled back to bytes; an output's image stride of a
// batch of one addresses nothing and may wrap.  Callers with a row-pitch limit apply it to L.row.
inline int check_layout(const void* base, uint64_t image, uint64_t row, uint64_t pixel, uint64_t chan, uint32_t n, uint32_t h, uint32_t w,
                        uint32_t chans, uint32_t elem, bool output, Layout& L)
{
    if ((uintptr_t)base % elem || image % elem || row % elem || pixel % elem || chan % elem) return FPNGB_ERR_ALIGNMENT;
    Layout E;
    if (!classify_layout(image / elem, row / elem, pixel / elem, chan / elem, n, h, w, chans, E)) return FPNGB_ERR_INVALID_ARG;
    if (output && !layout_disjoint(E, n, h, w, chans)) return FPNGB_ERR_INVALID_ARG;
    const uint64_t lim = UINT64_MAX / elem;
    if ((!output && E.image > lim) || E.row > lim || E.pixel > lim || E.chan > lim) return FPNGB_ERR_INVALID_ARG;
    L = Layout{E.image * elem, E.row * elem, E.pixel * elem, E.chan * elem, E.planar};
    uint64_t last = 0;
    if (!layout_span(base, L, n, h, w, chans, last) || last > UINT64_MAX - (uint64_t)(uintptr_t)base - (elem - 1)) return FPNGB_ERR_INVALID_ARG;
    return FPNGB_OK;
}

}  // namespace fpngb
