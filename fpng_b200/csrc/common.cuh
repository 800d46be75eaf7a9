// fpng_b200/csrc/common.cuh -- shared device/host definitions for the sm_90a fpng hot path.
//
// Vocabulary follows the reference (richgel999/fpng, src/fpng.cpp): scanlines/rows, filter bytes,
// literals, RLE matches, code books, zlib stream, IDAT.  Every kernel cites the reference lines whose
// behaviour it reproduces.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

namespace fpngb {

constexpr uint32_t kPngHeaderSize = 58;      // sig(8) IHDR(25) fdEC(17) IDAT len+type(8): fpng.cpp:1701,1770-1783
constexpr uint32_t kPngEncHeaderSize = 41;  // fpngb_encode_png_ragged_device's files: sig(8) IHDR(25) IDAT len+type(8), no fdEC
constexpr uint32_t kPngTrailerSize = 16;     // IDAT crc(4) + IEND(12): fpng.cpp:1794
constexpr uint32_t kZlibBitBase = kPngHeaderSize * 8;   // file-bit coordinate of zlib bit 0
constexpr uint32_t kAdlerMod = 65521;
constexpr uint32_t kMaxHdrBytes = 320;       // dynamic block header <= 2310 bits (fpng.cpp:798) + zlib hdr + BFINAL

// Per-image (2-pass) or shared (1-pass) Huffman code book in the form the kernels consume.
struct CodeBook {
    uint32_t lit[256];        // literal byte v: code | size << 16   (code already bit-reversed, LSB-first)
    uint32_t match[88];       // match of n pixels (n = 1..M): (len code | extra << size) | total_bits << 24
                              //   total_bits = size(len sym) + extra bits + 1 (the 1-bit distance code, always 0)
    uint32_t eob;             // symbol 256: code | size << 16
    uint32_t hdr_bits;        // number of valid bits in hdr[] (zlib hdr + BFINAL + BTYPE + dynamic header)
    uint8_t  lit_size[256];   // same sizes, byte form, for the counting kernel
    uint8_t  match_bits[88];  // total_bits per match length in pixels
    uint8_t  hdr[kMaxHdrBytes];
    uint8_t  sym_size[288];   // raw lit/len code sizes (used to build the decoder tables / tests)
    uint8_t  lit1_rule;       // RGBA 1-pass only: a one-pixel match can cost more than four literals under this table, so the
                              //   reference's check at fpng.cpp:1520-1528 is live (never with the shipped table)
    uint8_t  pad_[7];
};

// Per-image state produced by the offsets kernel and consumed by pack / checksum kernels.
struct ImageState {
    uint32_t zsize;           // zlib stream size in bytes (IDAT length)
    uint32_t stored;          // 1 -> stored-block fallback (fpng.cpp:1728-1758)
    uint32_t adler;           // Adler-32 of the filtered stream (compressed path)
    uint32_t crc_acc;         // XOR accumulator of tile CRC contributions
    uint32_t tiles_done;      // completion counter for the CRC tiles
    uint32_t last_unit_bits;  // bits of the last flush unit of the last row (capacity rule, SURVEY Q5)
    uint32_t status;          // 0 ok, nonzero = internal error
    uint32_t pad_;
};

// Deflate length code for a match of L bytes (3..258), RFC 1951 / fpng.cpp:498-512.
__host__ __device__ inline void deflate_len_code(uint32_t L, uint32_t& sym, uint32_t& xbits, uint32_t& xval)
{
    if (L >= 258) { sym = 285; xbits = 0; xval = 0; return; }
    uint32_t a = L - 3;
    if (a < 8) { sym = 257 + a; xbits = 0; xval = 0; return; }
    // groups of 4 symbols share an extra-bit count: xbits = floor(log2(a)) - 2
    uint32_t lg = 31 - (uint32_t)
#ifdef __CUDA_ARCH__
        __clz((int)a);
#else
        __builtin_clz(a);
#endif
    xbits = lg - 2;
    sym = 257 + 4 * xbits + 4 + ((a >> xbits) & 3);
    xval = a & ((1u << xbits) - 1);
}

// max pixels per match token: 255/3 and 252/4 (fpng.cpp:1052, 1212, 1330, 1506)
__host__ __device__ constexpr uint32_t max_match_pixels(uint32_t chans) { return chans == 3 ? 85u : 63u; }

// Worst-case file size: stored-block layout (fpng.cpp:1747) vs the compressed-path buffer (fpng.cpp:1705).
__host__ __device__ inline size_t max_encoded_size(uint32_t w, uint32_t h, uint32_t chans)
{
    size_t raw = ((size_t)w * chans + 1) * h;
    size_t stored = kPngHeaderSize + 6 + raw + 5 * ((raw + 65534) / 65535) + kPngTrailerSize;
    size_t comp = ((kPngHeaderSize + raw + 7) & ~(size_t)7) + kPngTrailerSize;
    return stored > comp ? stored : comp;
}

#define FPNGB_CUDA_OK(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) return (int)(1000 + (int)e__); } while (0)

}  // namespace fpngb
