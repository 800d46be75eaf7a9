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
// Outputs: w, h, chans (1 gray, 2 gray+alpha, 3, 4), idat_ofs = offset of the first IDAT chunk, idat_len = sum of the IDAT data
// lengths.  No byte at or beyond f[size] is read.
#pragma once
#include "container.cuh"

namespace fpngb {

#pragma nv_exec_check_disable
template <class Crc>
__host__ __device__ int png_walk(const uint8_t* f, uint32_t size, const Crc& crc, uint32_t* w, uint32_t* h, uint32_t* chans,
                                 uint32_t* idat_ofs, uint32_t* idat_len)
{
    *w = *h = *chans = 0; *idat_ofs = *idat_len = 0;
    if (size < 8 + 25 + 8 + 1 + 4 + 12) return FPNGB_DECODE_FAILED_NOT_PNG;
    if (!walk_tag(f, '\x89', 'P', 'N', 'G') || !walk_tag(f + 4, '\x0D', '\x0A', '\x1A', '\x0A')) return FPNGB_DECODE_FAILED_NOT_PNG;
    if (walk_be32(f + 8) != 13) return FPNGB_DECODE_FAILED_NOT_PNG;
    if (crc(f + 12, 17) != walk_be32(f + 29)) return FPNGB_DECODE_FAILED_HEADER_CRC32;
    *w = walk_be32(f + 16); *h = walk_be32(f + 20);
    if (!*w || !*h || *w > (1u << 24) || *h > (1u << 24)) return FPNGB_DECODE_FAILED_INVALID_DIMENSIONS;
    if ((uint64_t)*w * *h > (1u << 30)) return FPNGB_DECODE_FAILED_INVALID_DIMENSIONS;
    const uint32_t type = f[25];
    if (f[24] != 8 || f[26] || f[27] || f[28]) return FPNGB_DECODE_UNSUPPORTED_PNG;
    if (type == 0) *chans = 1; else if (type == 2) *chans = 3; else if (type == 4) *chans = 2; else if (type == 6) *chans = 4;
    else return FPNGB_DECODE_UNSUPPORTED_PNG;
    const bool gray = type == 0 || type == 4;
    bool in_idat = false, idat_done = false;
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
            if (in_idat) { in_idat = false; idat_done = true; }
            if (walk_tag(ty, 'I', 'H', 'D', 'R')) return FPNGB_DECODE_UNSUPPORTED_PNG;
            if (walk_tag(ty, 'P', 'L', 'T', 'E')) { if (gray) return FPNGB_DECODE_UNSUPPORTED_PNG; }
            else if (walk_tag(ty, 't', 'R', 'N', 'S')) { if (type == 0 || type == 2) return FPNGB_DECODE_UNSUPPORTED_PNG; }
            else if (!(ty[0] & 32)) return FPNGB_DECODE_UNSUPPORTED_PNG;      // unknown critical chunk
        }
        ofs += 8 + (size_t)len + 4;
    }
    if (!in_idat && !idat_done) return FPNGB_DECODE_FAILED_INVALID_IDAT;
    if (*idat_len < 2) return FPNGB_DECODE_FAILED_INVALID_IDAT;
    return FPNGB_DECODE_SUCCESS;
}

// The walk of the any-PNG calls: container_walk, and png_walk for the files it rejects with FPNGB_DECODE_NOT_FPNG.  *general is set
// when png_walk ran (whatever it returned).
#pragma nv_exec_check_disable
template <class Crc>
__host__ __device__ int any_png_walk(const uint8_t* f, uint32_t size, const Crc& crc, uint32_t* w, uint32_t* h, uint32_t* chans,
                                     uint32_t* idat_ofs, uint32_t* idat_len, bool* general)
{
    const int st = container_walk(f, size, crc, w, h, chans, idat_ofs, idat_len);
    *general = st == FPNGB_DECODE_NOT_FPNG;
    return *general ? png_walk(f, size, crc, w, h, chans, idat_ofs, idat_len) : st;
}

}  // namespace fpngb
