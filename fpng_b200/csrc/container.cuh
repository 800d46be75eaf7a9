// fpng_b200/csrc/container.cuh -- the PNG container walk, one function for the host and the device.
//
// PNG signature / IHDR / chunk walk with the reference's acceptance rules and return codes (fpng.cpp:2930-3077).
// Only chunk headers and the CRCs of the non-IDAT chunks are touched.  The host entry points (fpngb_get_info*,
// fpngb_decode_host, fpngb_decode_batch_host) instantiate it with host_crc32; container_walk_kernel
// (container_kernels.cu) with a byte-table CRC in constant memory, so both walks apply the same rules by construction.
// No byte at or beyond f[size] is ever read, whatever the length fields say.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include "../../include/fpng_b200.h"

namespace fpngb {

__host__ __device__ __forceinline__ uint32_t walk_be32(const uint8_t* p)
{
    return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}
__host__ __device__ __forceinline__ bool walk_tag(const uint8_t* t, char a, char b, char c, char d)
{
    return t[0] == (uint8_t)a && t[1] == (uint8_t)b && t[2] == (uint8_t)c && t[3] == (uint8_t)d;
}

// `crc(p, n)` returns the CRC-32 (PNG/zlib polynomial, fresh register) of the n bytes at p.
#pragma nv_exec_check_disable
template <class Crc>
__host__ __device__ int container_walk(const uint8_t* f, uint32_t size, const Crc& crc, uint32_t* w, uint32_t* h, uint32_t* chans,
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
    if (f[26] || f[27] || f[28] || f[24] != 8) return FPNGB_DECODE_NOT_FPNG;
    if (f[25] == 2) *chans = 3; else if (f[25] == 6) *chans = 4;
    if (!*chans) return FPNGB_DECODE_NOT_FPNG;
    bool have_fdec = false;
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
        const uint8_t* d = f + ofs + 8;
        if (walk_tag(ty, 'I', 'E', 'N', 'D')) break;
        if (is_idat) {
            if (*idat_ofs || !have_fdec) return FPNGB_DECODE_NOT_FPNG;
            *idat_ofs = (uint32_t)ofs; *idat_len = len;
            if (len < 7) return FPNGB_DECODE_FAILED_INVALID_IDAT;
        } else if (walk_tag(ty, 'f', 'd', 'E', 'C')) {
            if (have_fdec || len != 5) return FPNGB_DECODE_NOT_FPNG;
            if (d[0] != 82 || d[1] != 36 || d[2] != 147 || d[3] != 227 || d[4] != 0) return FPNGB_DECODE_NOT_FPNG;
            have_fdec = true;
        } else if (!(ty[0] & 32)) return FPNGB_DECODE_NOT_FPNG;
        ofs += 8 + (size_t)len + 4;
    }
    if (!have_fdec || !*idat_ofs) return FPNGB_DECODE_NOT_FPNG;
    return FPNGB_DECODE_SUCCESS;
}

}  // namespace fpngb
