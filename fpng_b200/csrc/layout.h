// fpng_b200/csrc/layout.h -- the pixel layouts of the strided device entry points (include/fpng_b200.h, "Pixel layouts").
// A batch is an [n, h, w, chans] array of bytes: byte (i, y, x, c) at base + i*image + y*row + x*pixel + c*chan.
#pragma once
#include <stddef.h>
#include <stdint.h>

namespace fpngb {

struct Layout {
    uint64_t image, row, pixel, chan;   // byte strides after canonicalisation
    bool planar;                        // pixel == 1 (one byte plane per channel); else interleaved: pixel == chans, chan == 1
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

}  // namespace fpngb
