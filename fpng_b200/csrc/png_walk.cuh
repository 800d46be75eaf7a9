// fpng_b200/csrc/png_walk.cuh -- the container walk of general PNG files, one function for the host and the device.
//
// png_walk accepts the 8-bit, non-interlaced gray, gray+alpha, RGB and RGBA files of any writer (libpng, PIL, OpenCV, ...), the
// files the general decode (inflate_kernels.cu, png_unfilter_kernels.cu) reads.  It runs only where container_walk (container.cuh)
// returned FPNGB_DECODE_NOT_FPNG: fpng-written files keep container_walk's row.  Signature, IHDR, dimension limits, chunk framing
// and the CRCs of the non-IDAT chunks are checked with container_walk's rules and codes; then:
//   * IHDR other than bit depth 8, color type 0 / 2 / 4 / 6, compression 0, filter method 0, interlace 0: FPNGB_DECODE_UNSUPPORTED_PNG
//     (palette, 16-bit, sub-byte depths, Adam7);
//   * a critical chunk other than IHDR / PLTE / IDAT / IEND, a second IHDR, a PLTE in a gray file, or a tRNS chunk in a color type 0
//     or 2 file (its transparent color would need an alpha channel the file does not have): FPNGB_DECODE_UNSUPPORTED_PNG.  A PLTE
//     in an RGB / RGBA file is a suggested palette and ignored, as are all other ancillary chunks;
//   * the IDAT chunks must be consecutive (FAILED_CHUNK_PARSING otherwise); zero-length ones are legal.  No IDAT, or fewer than 2
//     data bytes in all: FAILED_INVALID_IDAT.
// With flags & FPNGB_PNG_ALL_FORMATS the walk also accepts every other format PNG defines (include/fpng_b200.h lists the rules):
//   * IHDR (color type: depths) 0: 1 2 4 8 16, 2: 8 16, 3: 1 2 4 8, 4: 8 16, 6: 8 16, interlace 0 or 1; anything else is still
//     FPNGB_DECODE_UNSUPPORTED_PNG;
//   * color type 3 needs exactly one PLTE before the first IDAT, 1..256 entries (length a nonzero multiple of 3, <= 768);
//   * tRNS in color types 0 / 2 / 3: at most one, before the first IDAT, after PLTE in type 3; length 2 (type 0), 6 (type 2), at
//     most the palette's entries (type 3).  tRNS in types 4 / 6 is ignored, as without the flag.
//   Violations of the PLTE and tRNS rules give FAILED_CHUNK_PARSING.  *fm (PngFormat) describes the file for the decode kernels.
// Outputs: w, h, chans (1 gray, 2 gray+alpha, 3, 4; with the flag, +1 for a tRNS chunk in types 0 / 2 / 3 and 3 for palette files),
// idat_ofs = offset of the first IDAT chunk, idat_len = sum of the IDAT data lengths.  No byte at or beyond f[size] is read.
#pragma once
#include "container.cuh"

namespace fpngb {

// What the decode kernels need beyond the info row (png_walk with FPNGB_PNG_ALL_FORMATS; zero for other files).
struct PngFormat {
    uint32_t depth, type, interlace;        // IHDR bit depth, color type, interlace method
    uint32_t plte_ofs, plte_n;              // file offset of the PLTE data and its entry count (color type 3)
    uint32_t trns_ofs, trns_len;            // file offset of the tRNS data and its length (types 0 / 2 / 3; trns_ofs 0: no tRNS)
    uint32_t ext;                           // 1: a file the 8-bit kernels do not read (depth != 8, Adam7, palette or a color key)
    unsigned long long raw_len;             // inflated bytes: every row of every pass with its filter byte (png_raw_len)
};

// Adam7 (PNG spec 8.2): pass k takes the pixels x = x0 + i * dx, y = y0 + j * dy.  Nibble k of each constant is pass k's value
// (x0 0 4 0 2 0 1 0, y0 0 0 4 0 2 0 1, dx 8 8 4 4 2 2 1, dy 8 8 8 4 4 2 2), so a run-time k needs no table in local memory.
__host__ __device__ __forceinline__ void adam7_pass(uint32_t k, uint32_t* x0, uint32_t* y0, uint32_t* dx, uint32_t* dy)
{
    *x0 = (0x0102040u >> (4 * k)) & 15u; *y0 = (0x1020400u >> (4 * k)) & 15u;
    *dx = (0x1224488u >> (4 * k)) & 15u; *dy = (0x2244888u >> (4 * k)) & 15u;
}
// pixels of pass k of a w x h image along one axis: ceil((n - o) / d), 0 when n <= o
__host__ __device__ __forceinline__ uint32_t pass_extent(uint32_t n, uint32_t o, uint32_t d) { return n > o ? (n - o + d - 1) / d : 0u; }

// Inflated size of a w x h file with bits per pixel `bits`: h * (1 + ceil(w * bits / 8)) for interlace 0, the sum of that expression
// over the 7 Adam7 passes (an empty pass has no rows and no filter bytes) for interlace 1.  64 bits: 16-bit RGBA at 2^30 pixels
// passes 4 GiB.
__host__ __device__ __forceinline__ unsigned long long png_raw_len(uint32_t w, uint32_t h, uint32_t bits, uint32_t interlace)
{
    if (!interlace) return (unsigned long long)h * (1ull + ((unsigned long long)w * bits + 7) / 8);
    unsigned long long n = 0;
    for (uint32_t k = 0; k < 7; k++) {
        uint32_t x0, y0, dx, dy;
        adam7_pass(k, &x0, &y0, &dx, &dy);
        const uint32_t pw = pass_extent(w, x0, dx), ph = pass_extent(h, y0, dy);
        if (pw && ph) n += (unsigned long long)ph * (1ull + ((unsigned long long)pw * bits + 7) / 8);
    }
    return n;
}

#pragma nv_exec_check_disable
template <class Crc>
__host__ __device__ int png_walk(const uint8_t* f, uint32_t size, const Crc& crc, uint32_t flags, uint32_t* w, uint32_t* h,
                                 uint32_t* chans, uint32_t* idat_ofs, uint32_t* idat_len, PngFormat* fm)
{
    *w = *h = *chans = 0; *idat_ofs = *idat_len = 0;
    *fm = PngFormat{};
    if (size < 8 + 25 + 8 + 1 + 4 + 12) return FPNGB_DECODE_FAILED_NOT_PNG;
    if (!walk_tag(f, '\x89', 'P', 'N', 'G') || !walk_tag(f + 4, '\x0D', '\x0A', '\x1A', '\x0A')) return FPNGB_DECODE_FAILED_NOT_PNG;
    if (walk_be32(f + 8) != 13) return FPNGB_DECODE_FAILED_NOT_PNG;
    if (crc(f + 12, 17) != walk_be32(f + 29)) return FPNGB_DECODE_FAILED_HEADER_CRC32;
    *w = walk_be32(f + 16); *h = walk_be32(f + 20);
    if (!*w || !*h || *w > (1u << 24) || *h > (1u << 24)) return FPNGB_DECODE_FAILED_INVALID_DIMENSIONS;
    if ((uint64_t)*w * *h > (1u << 30)) return FPNGB_DECODE_FAILED_INVALID_DIMENSIONS;
    const uint32_t type = f[25], depth = f[24];
    const bool all = (flags & FPNGB_PNG_ALL_FORMATS) != 0;
    if (!all) {
        if (depth != 8 || f[26] || f[27] || f[28]) return FPNGB_DECODE_UNSUPPORTED_PNG;
    } else {
        if (f[26] || f[27] || f[28] > 1) return FPNGB_DECODE_UNSUPPORTED_PNG;
        const bool d8 = depth == 8, d16 = depth == 16, sub = depth == 1 || depth == 2 || depth == 4;
        if (!((type == 0 && (sub || d8 || d16)) || (type == 3 && (sub || d8)) || ((type == 2 || type == 4 || type == 6) && (d8 || d16))))
            return FPNGB_DECODE_UNSUPPORTED_PNG;
    }
    uint32_t samples;
    if (type == 0) *chans = samples = 1; else if (type == 2) *chans = samples = 3; else if (type == 4) *chans = samples = 2;
    else if (type == 6) *chans = samples = 4; else if (type == 3 && all) { *chans = 3; samples = 1; }
    else return FPNGB_DECODE_UNSUPPORTED_PNG;
    const bool gray = type == 0 || type == 4;
    bool in_idat = false, idat_done = false, trns = false;
    size_t ofs = 33;
    for (;;) {
        if (ofs >= size || size - ofs < 12) return FPNGB_DECODE_FAILED_CHUNK_PARSING;
        const uint32_t len = walk_be32(f + ofs);
        if ((uint64_t)ofs + 8 + len + 4 > size) return FPNGB_DECODE_FAILED_CHUNK_PARSING;
        const uint8_t* ty = f + ofs + 4;
        for (int i = 0; i < 4; i++) {
            const bool up = ty[i] >= 65 && ty[i] <= 90, lo = ty[i] >= 97 && ty[i] <= 122;
            if (!up && !lo) return FPNGB_DECODE_FAILED_CHUNK_PARSING;
        }
        const bool is_idat = walk_tag(ty, 'I', 'D', 'A', 'T');
        if (!is_idat && crc(ty, 4 + (size_t)len) != walk_be32(f + ofs + 8 + len)) return FPNGB_DECODE_FAILED_HEADER_CRC32;
        if (walk_tag(ty, 'I', 'E', 'N', 'D')) break;
        if (is_idat) {
            if (idat_done) return FPNGB_DECODE_FAILED_CHUNK_PARSING;             // a second run of IDAT chunks
            if (!in_idat) *idat_ofs = (uint32_t)ofs;
            in_idat = true;
            *idat_len += len;                                                   // <= size: every chunk lies inside the file
        } else {
            const bool after_idat = in_idat || idat_done;
            if (in_idat) { in_idat = false; idat_done = true; }
            if (walk_tag(ty, 'I', 'H', 'D', 'R')) return FPNGB_DECODE_UNSUPPORTED_PNG;
            if (walk_tag(ty, 'P', 'L', 'T', 'E')) {
                if (gray) return FPNGB_DECODE_UNSUPPORTED_PNG;
                if (type == 3) {
                    if (fm->plte_n || after_idat || !len || len % 3 || len > 768) return FPNGB_DECODE_FAILED_CHUNK_PARSING;
                    fm->plte_ofs = (uint32_t)ofs + 8; fm->plte_n = len / 3;
                }
            } else if (walk_tag(ty, 't', 'R', 'N', 'S')) {
                if (type == 0 || type == 2 || type == 3) {
                    if (!all) return FPNGB_DECODE_UNSUPPORTED_PNG;
                    if (trns || after_idat) return FPNGB_DECODE_FAILED_CHUNK_PARSING;
                    if (type == 0 ? len != 2 : type == 2 ? len != 6 : (!fm->plte_n || len > fm->plte_n)) return FPNGB_DECODE_FAILED_CHUNK_PARSING;
                    trns = true; fm->trns_ofs = (uint32_t)ofs + 8; fm->trns_len = len;
                }
            } else if (!(ty[0] & 32)) return FPNGB_DECODE_UNSUPPORTED_PNG;      // unknown critical chunk
        }
        ofs += 8 + (size_t)len + 4;
    }
    if (type == 3 && !fm->plte_n) return FPNGB_DECODE_FAILED_CHUNK_PARSING;
    if (!in_idat && !idat_done) return FPNGB_DECODE_FAILED_INVALID_IDAT;
    if (*idat_len < 2) return FPNGB_DECODE_FAILED_INVALID_IDAT;
    if (all) {
        if (trns) *chans += 1;
        fm->depth = depth; fm->type = type; fm->interlace = f[28];
        fm->ext = depth != 8 || f[28] || type == 3 || trns;
        fm->raw_len = png_raw_len(*w, *h, depth * samples, f[28]);
    }
    return FPNGB_DECODE_SUCCESS;
}

// The walk of the any-PNG calls: container_walk, and png_walk for the files it rejects with FPNGB_DECODE_NOT_FPNG.  *general is set
// when png_walk ran (whatever it returned).
#pragma nv_exec_check_disable
template <class Crc>
__host__ __device__ int any_png_walk(const uint8_t* f, uint32_t size, const Crc& crc, uint32_t flags, uint32_t* w, uint32_t* h,
                                     uint32_t* chans, uint32_t* idat_ofs, uint32_t* idat_len, bool* general, PngFormat* fm)
{
    *fm = PngFormat{};
    const int st = container_walk(f, size, crc, w, h, chans, idat_ofs, idat_len);
    *general = st == FPNGB_DECODE_NOT_FPNG;
    return *general ? png_walk(f, size, crc, flags, w, h, chans, idat_ofs, idat_len, fm) : st;
}

}  // namespace fpngb
