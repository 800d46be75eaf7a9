// fpng_b200/csrc/crc_math.cuh -- CRC-32 in one place: the polynomial, its byte table, GF(2) arithmetic modulo it, the
// host builders of every CRC table the kernels upload, and the device helpers those kernels share.  Values are in the
// reflected representation of the IEEE 802.3 CRC (fpng.cpp:195-249): bit 31 is the coefficient of x^0, so "1" is
// 0x80000000 and "x" is 0x40000000.  Advancing a CRC register over n zero bytes is the multiplication by x^(8n); NVIDIA
// GPUs have no carry-less multiply (the reference folds with PCLMULQDQ, fpng.cpp:255-281).
//
// The library compiles without -rdc, so every translation unit keeps its own __device__ / __constant__ copy of the tables
// it reads; only their contents come from here.
#pragma once
#include <stdint.h>

namespace fpngb {

constexpr uint32_t kCrcPoly = 0xEDB88320u;          // reflected IEEE 802.3 (fpng.cpp:195-249)
constexpr uint32_t kCrcOne = 0x80000000u;           // the polynomial "1" in reflected form

__host__ __device__ constexpr uint32_t gf2_mulmod(uint32_t a, uint32_t b)
{
    uint32_t p = 0;
#pragma unroll 8
    for (int i = 0; i < 32; i++) {
        p ^= (a & (0x80000000u >> i)) ? b : 0u;
        b = (b >> 1) ^ ((b & 1u) ? kCrcPoly : 0u);
    }
    return p;
}

__device__ inline uint32_t gf2_pow(const uint32_t* tab, unsigned long long e)
{
    uint32_t r = kCrcOne;
    for (int k = 0; e; k++, e >>= 1)
        if (e & 1ull) r = gf2_mulmod(r, tab[k]);
    return r;
}

// byte table: t[n] is the register after byte n from a zero register
struct CrcByteTable { uint32_t t[256]; };
constexpr CrcByteTable crc_byte_table()
{
    CrcByteTable r{};
    for (uint32_t n = 0; n < 256; n++) {
        uint32_t c = n;
        for (int k = 0; k < 8; k++) c = (c & 1u) ? (kCrcPoly ^ (c >> 1)) : (c >> 1);
        r.t[n] = c;
    }
    return r;
}
static_assert(crc_byte_table().t[1] == 0x77073096u, "CRC-32 byte table");
static_assert([] {
    const CrcByteTable t = crc_byte_table();
    uint32_t c = 0xFFFFFFFFu;
    for (const char* s = "123456789"; *s; s++) c = t.t[(c ^ (uint8_t)*s) & 0xFFu] ^ (c >> 8);
    return ~c;
}() == 0xCBF43926u, "CRC-32 check value");

// ---- host builders of the kernels' tables ----------------------------------------------------------------------------------

// x^e mod P
inline uint32_t xpow(unsigned long long e)
{
    uint32_t r = kCrcOne, s = kCrcOne >> 1;
    for (; e; e >>= 1, s = gf2_mulmod(s, s))
        if (e & 1ull) r = gf2_mulmod(r, s);
    return r;
}

// xp[k] = x^(2^k) mod P: the table gf2_pow reads
inline void crc_xpow2_table(uint32_t xp[64])
{
    xp[0] = kCrcOne >> 1;
    for (int k = 1; k < 64; k++) xp[k] = gf2_mulmod(xp[k - 1], xp[k - 1]);
}

// slice-by-4: t[k][n] is the register after byte n followed by k zero bytes
inline void crc_slice4_tables(uint32_t t[4][256])
{
    const CrcByteTable b = crc_byte_table();
    for (uint32_t n = 0; n < 256; n++) t[0][n] = b.t[n];
    for (uint32_t n = 0; n < 256; n++) for (int k = 1; k < 4; k++) t[k][n] = (t[k - 1][n] >> 8) ^ t[0][t[k - 1][n] & 0xFF];
}

// f[k][n]: byte k (= n) of (reg ^ word) advanced over `bytes` >= 4 bytes.  The word update
// "reg = f[0][b0] ^ f[1][b1] ^ f[2][b2] ^ f[3][b3]" is slice-by-4's 4-byte step followed by x^(8 * (bytes - 4)).
inline void crc_advance_tables(uint32_t f[4][256], unsigned long long bytes)
{
    uint32_t t[4][256];
    crc_slice4_tables(t);
    const uint32_t adv = xpow(8ull * (bytes - 4));
    for (int k = 0; k < 4; k++) for (uint32_t n = 0; n < 256; n++) f[k][n] = gf2_mulmod(t[3 - k][n], adv);
}

// nibble table of the multiplication by c: m[j][n] = (n << 4j) * c, so a * c is the XOR of m[j][nibble j of a] (mul_nibbles)
inline void crc_mul_table(uint32_t m[8][16], uint32_t c)
{
    for (int j = 0; j < 8; j++) for (uint32_t n = 0; n < 16; n++) m[j][n] = gf2_mulmod(n << (4 * j), c);
}

// ---- device helpers ----------------------------------------------------------------------------------------------------------

// a * c through the nibble table crc_mul_table(t, c) built (GF(2)-linear in a)
__device__ __forceinline__ uint32_t mul_nibbles(const uint32_t (*t)[16], uint32_t a)
{
    uint32_t r = __ldg(&t[0][a & 15u]);
#pragma unroll
    for (int j = 1; j < 8; j++) r ^= __ldg(&t[j][(a >> (4 * j)) & 15u]);
    return r;
}

// the register after the nbits low bits of v, least significant first: the order Deflate packs bits and the reflected CRC reads them
__device__ __forceinline__ uint32_t crc_bits(uint32_t reg, uint32_t v, uint32_t nbits)
{
    for (uint32_t i = 0; i < nbits; i++) { reg = (reg >> 1) ^ (((reg ^ (v >> i)) & 1u) ? kCrcPoly : 0u); }
    return reg;
}
__device__ __forceinline__ uint32_t crc_bit_step(uint32_t reg, uint32_t bit) { return crc_bits(reg, bit, 1); }

}  // namespace fpngb
