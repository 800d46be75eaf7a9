// fpng_b200/csrc/checksum_kernels.cu -- CRC-32 of the IDAT chunk on the device.
//
// The reference folds with PCLMULQDQ (fpng.cpp:255-281) or slices by 4 (fpng.cpp:234-249).  NVIDIA GPUs have no
// carry-less multiply, so the same GF(2) algebra is done as
//   * per-thread slice-by-4 table CRC of a 128-byte chunk staged in shared memory (conflict-free padded layout),
//   * a tree of "multiply by x^(8*len) mod P" combines (32-step shift/xor products) inside the CTA,
//   * Horner accumulation over the CTA's consecutive 32 KiB tiles, one modular power per CTA, an XOR-reduce over
//     CTAs in global memory, and a last-CTA-done finaliser that writes the big-endian CRC (fpng.cpp:1797-1800).
// The message ("IDAT" + zlib stream = file bytes [54, 58+zsize)) is treated as zero-padded to a tile boundary;
// the padding is undone with x^(-8*pad).  Pre/post conditioning (init/xorout 0xFFFFFFFF) is the usual
// "invert the first four message bytes, invert the result".
#include "kernels.cuh"
#include "crc_math.cuh"
#include <string.h>

namespace fpngb {

constexpr int kCrcThreads = 256;
constexpr int kChunkWords = 32;                     // 128 bytes per thread
constexpr int kTileWords = kCrcThreads * kChunkWords;
constexpr uint32_t kTileBytes = kTileWords * 4;     // 32 KiB
constexpr int kTilesPerCta = 8;

__constant__ uint32_t c_xpow2[64];                  // x^(2^k) mod P
__constant__ uint32_t c_xinvpow2[64];               // x^-(2^k) mod P
__constant__ uint32_t c_level[8];                   // x^(8 * 128 * 2^k): chunk-combine multipliers
__constant__ uint32_t c_tile;                       // x^(8 * kTileBytes)
__device__ uint32_t g_crc_tables[4][256];           // slice-by-4
__device__ uint32_t g_crc_mul[8][8][16];            // g_crc_mul[k][j][n] = (n << 4j) * x^(8*128*2^k) mod P: multiply-by-constant as 8 nibble lookups

static uint32_t h_tables[4][256];
static bool h_tables_ready = false;

static void host_tables()
{
    if (h_tables_ready) return;
    for (uint32_t n = 0; n < 256; n++) {
        uint32_t c = n;
        for (int k = 0; k < 8; k++) c = (c & 1) ? (kCrcPoly ^ (c >> 1)) : (c >> 1);
        h_tables[0][n] = c;
    }
    for (uint32_t n = 0; n < 256; n++)
        for (int t = 1; t < 4; t++) h_tables[t][n] = (h_tables[t - 1][n] >> 8) ^ h_tables[0][h_tables[t - 1][n] & 0xFF];
    h_tables_ready = true;
}

uint32_t host_crc32(const void* data, size_t n, uint32_t prev)
{
    host_tables();
    const uint8_t* p = (const uint8_t*)data;
    uint32_t c = ~prev;
    for (size_t i = 0; i < n; i++) c = h_tables[0][(c ^ p[i]) & 0xFF] ^ (c >> 8);
    return ~c;
}

int checksum_tables_init()
{
    host_tables();
    uint32_t xp[64], xi[64], lvl[8];
    xp[0] = 0x40000000u; xi[0] = kCrcXInv;
    for (int k = 1; k < 64; k++) { xp[k] = gf2_mulmod(xp[k - 1], xp[k - 1]); xi[k] = gf2_mulmod(xi[k - 1], xi[k - 1]); }
    // x^(8*128*2^k) = x^(2^(10+k))
    for (int k = 0; k < 8; k++) lvl[k] = xp[10 + k];
    const uint32_t tile = xp[18];                   // 8 * 32768 = 2^18
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(c_xpow2, xp, sizeof xp));
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(c_xinvpow2, xi, sizeof xi));
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(c_level, lvl, sizeof lvl));
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(c_tile, &tile, sizeof tile));
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(g_crc_tables, h_tables, sizeof h_tables));
    static uint32_t mul[8][8][16];
    for (int k = 0; k < 8; k++) for (int j = 0; j < 8; j++) for (uint32_t n = 0; n < 16; n++) mul[k][j][n] = gf2_mulmod(n << (4 * j), lvl[k]);
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(g_crc_mul, mul, sizeof mul));
    return 0;
}

// Mask selecting the bytes of the little-endian word at file offset wo that lie in [lo, hi).
__device__ __forceinline__ uint32_t byte_range_mask(uint32_t wo, uint32_t lo, uint32_t hi)
{
    const uint32_t a = max(wo, lo), b = min(wo + 4u, hi);
    if (a >= b) return 0u;
    return (0xFFFFFFFFu << (8u * (a - wo))) & (0xFFFFFFFFu >> (8u * (wo + 4u - b)));
}

// Word of the conditioned, zero-padded message at buffer offset wo (wo % 4 == 0): bytes outside [start, L) read
// as zero, the first four message bytes are XORed with the (little-endian) initial register value.
__device__ __forceinline__ uint32_t condition_word(uint32_t v, uint32_t wo, uint32_t start, uint32_t L, uint32_t init)
{
    const uint32_t keep = byte_range_mask(wo, start, L);
    const uint32_t pat = wo <= start ? ((start - wo) < 4u ? (init << (8u * (start - wo))) : 0u)
                                      : ((wo - start) < 4u ? (init >> (8u * (wo - start))) : 0u);
    const uint32_t inv = byte_range_mask(wo, start, start + 4u) & pat;
    return (v ^ inv) & keep;
}

// a * x^(8*128*2^k) mod P through the level's nibble tables (GF(2)-linear in a)
__device__ __forceinline__ uint32_t mul_level(const uint32_t (*t)[16], uint32_t a)
{
    uint32_t r = t[0][a & 15u];
#pragma unroll
    for (int j = 1; j < 8; j++) r ^= t[j][(a >> (4 * j)) & 15u];
    return r;
}

__global__ void __launch_bounds__(kCrcThreads) idat_crc_kernel(CrcParams p)
{
    __shared__ uint32_t s_tab[4][256];
    __shared__ uint32_t s_mul[8][8][16];
    __shared__ uint32_t s_data[kCrcThreads * (kChunkWords + 1)];
    __shared__ uint32_t s_warp[kCrcThreads / 32];

    const uint32_t img = blockIdx.y, b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    ImageState* st = p.st + img;
    if (p.stored_only && !st->stored) return;
    const uint32_t L = kPngHeaderSize + st->zsize;                      // end of the CRC'd region (buffer offset)
    const uint32_t start = p.msg_start, init = p.init_xor;
    const uint32_t ntiles = (L + kTileBytes - 1) / kTileBytes;
    const uint32_t nctas = (ntiles + kTilesPerCta - 1) / kTilesPerCta;
    if (b >= nctas) return;

    for (uint32_t i = tid; i < 1024; i += blockDim.x) { (&s_tab[0][0])[i] = (&g_crc_tables[0][0])[i]; (&s_mul[0][0][0])[i] = (&g_crc_mul[0][0][0])[i]; }

    const uint8_t* file = p.out + (size_t)img * p.out_stride;
    const uint32_t t0 = b * kTilesPerCta, t1 = min(t0 + kTilesPerCta, ntiles);
    uint32_t acc = 0;                                                  // Horner accumulator (thread 0)

    for (uint32_t tile = t0; tile < t1; tile++) {
        const uint32_t tile_ofs = tile * kTileBytes;
        __syncthreads();
        // coalesced 16-byte loads -> padded shared layout (chunk c at words [33c, 33c+32))
        // tiles strictly inside the message need no conditioning (only the first and last tile of a file do)
        const bool interior = tile_ofs >= start + 4u && tile_ofs + kTileBytes <= L;
        for (uint32_t g = tid; g < kTileWords / 4; g += blockDim.x) {
            const uint32_t wo = tile_ofs + g * 16u;
            const uint32_t wi = g * 4u, base = (wi / kChunkWords) * (kChunkWords + 1) + (wi % kChunkWords);
            if (interior) {
                const uint4 v = *reinterpret_cast<const uint4*>(file + wo);
                s_data[base + 0] = v.x; s_data[base + 1] = v.y; s_data[base + 2] = v.z; s_data[base + 3] = v.w;
            } else {
                uint4 v = make_uint4(0, 0, 0, 0);
                if (wo < L) v = *reinterpret_cast<const uint4*>(file + wo);
                s_data[base + 0] = condition_word(v.x, wo, start, L, init);
                s_data[base + 1] = condition_word(v.y, wo + 4u, start, L, init);
                s_data[base + 2] = condition_word(v.z, wo + 8u, start, L, init);
                s_data[base + 3] = condition_word(v.w, wo + 12u, start, L, init);
            }
        }
        __syncthreads();

        uint32_t crc = 0;
        const uint32_t* chunk = s_data + tid * (kChunkWords + 1);
#pragma unroll 4
        for (int j = 0; j < kChunkWords; j++) {
            const uint32_t x = chunk[j] ^ crc;
            crc = s_tab[3][x & 0xFF] ^ s_tab[2][(x >> 8) & 0xFF] ^ s_tab[1][(x >> 16) & 0xFF] ^ s_tab[0][x >> 24];
        }
        // tree combine: chunk i must be multiplied by x^(8*128*(255-i))
#pragma unroll
        for (int k = 0; k < 5; k++) {
            const uint32_t right = __shfl_down_sync(0xFFFFFFFFu, crc, 1u << k);
            const uint32_t prod = mul_level(s_mul[k], crc);
            if ((lane & ((2u << k) - 1u)) == 0) crc = prod ^ right;
        }
        if (lane == 0) s_warp[warp] = crc;
        __syncthreads();
        if (warp == 0) {
            uint32_t v = lane < kCrcThreads / 32 ? s_warp[lane] : 0u;
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const uint32_t right = __shfl_down_sync(0xFFFFFFFFu, v, 1u << k);
                const uint32_t prod = mul_level(s_mul[5 + k], v);
                if ((lane & ((2u << k) - 1u)) == 0) v = prod ^ right;
            }
            if (lane == 0) acc = gf2_mulmod(acc, c_tile) ^ v;
        }
    }

    if (tid == 0) {
        // shift the CTA's value to the padded end, fold into the image accumulator
        const unsigned long long tail_bytes = (unsigned long long)(ntiles - t1) * kTileBytes;
        acc = gf2_mulmod(acc, gf2_pow(c_xpow2, tail_bytes * 8ull));
        atomicXor(&st->crc_acc, acc);
        __threadfence();
        const uint32_t done = atomicAdd(&st->tiles_done, 1u);
        if (done == nctas - 1) {
            __threadfence();
            const uint32_t total = atomicXor(&st->crc_acc, 0u);
            const unsigned long long pad = (unsigned long long)ntiles * kTileBytes - L;
            const uint32_t crc = gf2_mulmod(total, gf2_pow(c_xinvpow2, pad * 8ull)) ^ 0xFFFFFFFFu;
            uint8_t* q = p.out + (size_t)img * p.out_stride + L;
            q[0] = (uint8_t)(crc >> 24); q[1] = (uint8_t)(crc >> 16); q[2] = (uint8_t)(crc >> 8); q[3] = (uint8_t)crc;
        }
    }
}

void launch_crc(const CrcParams& p, uint32_t n, cudaStream_t s)
{
    dim3 grid(p.max_tiles, n);
    idat_crc_kernel<<<grid, kCrcThreads, 0, s>>>(p);
}

// Adler-32 partials of a flat device buffer: CTA c covers bytes [c*64Ki, +64Ki) and writes (S1, S2) mod 65521 where
// S1 = sum x_i and S2 = sum (len - i) x_i over its chunk; the host folds the chunks with a' = a + S1, b' = b + len*a + S2
// (the same recurrence fpng.cpp:403-487 evaluates byte by byte).
constexpr uint32_t kAdlerChunk = 65536;
__global__ void __launch_bounds__(256) adler_buffer_kernel(const uint8_t* __restrict__ buf, size_t n, uint2* __restrict__ partials)
{
    __shared__ unsigned long long s_a[8], s_b[8];
    const size_t c0 = (size_t)blockIdx.x * kAdlerChunk;
    const uint32_t len = (uint32_t)min((size_t)kAdlerChunk, n - c0);
    unsigned long long A = 0, B = 0;
    for (uint32_t i = threadIdx.x * 16u; i < len; i += blockDim.x * 16u) {
        uint32_t wd[4] = {0, 0, 0, 0};
        if (i + 16u <= len) { const uint4 v = *reinterpret_cast<const uint4*>(buf + c0 + i); wd[0] = v.x; wd[1] = v.y; wd[2] = v.z; wd[3] = v.w; }
        else for (uint32_t k = 0; i + k < len; k++) wd[k >> 2] |= (uint32_t)buf[c0 + i + k] << (8 * (k & 3));
        uint32_t t1 = 0, t2 = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) { t1 = __dp4a(wd[k], 0x01010101u, t1); t2 = __dp4a(wd[k], 0x03020100u + 0x04040404u * k, t2); }
        A += t1; B += (unsigned long long)i * t1 + t2;
    }
    for (int o = 16; o > 0; o >>= 1) { A += __shfl_xor_sync(0xFFFFFFFFu, A, o); B += __shfl_xor_sync(0xFFFFFFFFu, B, o); }
    if ((threadIdx.x & 31) == 0) { s_a[threadIdx.x >> 5] = A; s_b[threadIdx.x >> 5] = B; }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long a = 0, b = 0;
        for (int i = 0; i < 8; i++) { a += s_a[i]; b += s_b[i]; }
        partials[blockIdx.x] = make_uint2((uint32_t)(a % kAdlerMod), (uint32_t)(((unsigned long long)len * a - b) % kAdlerMod));
    }
}

uint32_t adler_chunk_bytes() { return kAdlerChunk; }
void launch_adler_buffer(const uint8_t* d_buf, size_t n, uint2* d_partials, cudaStream_t s)
{
    const uint32_t nchunks = (uint32_t)((n + kAdlerChunk - 1) / kAdlerChunk);
    adler_buffer_kernel<<<nchunks, 256, 0, s>>>(d_buf, n, d_partials);
}

uint32_t crc_ctas_for(size_t max_file_bytes)
{
    const size_t ntiles = (max_file_bytes + kTileBytes - 1) / kTileBytes;
    return (uint32_t)((ntiles + kTilesPerCta - 1) / kTilesPerCta);
}

}  // namespace fpngb

// ------------------------------------------------------------------------------------------------
// Compaction of a batch of encoded files (fixed stride, variable size) into one contiguous device buffer, each file
// starting 16-byte aligned: the staging step before the NCCL gather of a rank's shard (fpng_b200/dist.py).
// ------------------------------------------------------------------------------------------------
namespace fpngb {

__global__ void __launch_bounds__(1024) compact_offsets_kernel(const uint32_t* __restrict__ sizes, uint32_t n, unsigned long long* __restrict__ offsets)
{
    __shared__ unsigned long long s_warp[32];
    __shared__ unsigned long long s_base;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_base = 0;
    __syncthreads();
    for (uint32_t i0 = 0; i0 < n; i0 += blockDim.x) {
        const uint32_t i = i0 + tid;
        const unsigned long long v = i < n ? (((unsigned long long)sizes[i] + 15ull) & ~15ull) : 0ull;
        unsigned long long s = v;
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long u = __shfl_up_sync(0xFFFFFFFFu, s, o); if (lane >= (uint32_t)o) s += u; }
        if (lane == 31) s_warp[warp] = s;
        __syncthreads();
        unsigned long long wb = 0, tot = 0;
        for (uint32_t k = 0; k < blockDim.x / 32; k++) { if (k < warp) wb += s_warp[k]; tot += s_warp[k]; }
        if (i < n) offsets[i] = s_base + wb + s - v;
        __syncthreads();
        if (tid == 0) s_base += tot;
        __syncthreads();
    }
    if (tid == 0) offsets[n] = s_base;
}

// file f at files + src_offsets[f], or at files + f * stride when src_offsets is null
__global__ void __launch_bounds__(256) compact_copy_kernel(const uint8_t* __restrict__ files, size_t stride, const uint32_t* __restrict__ sizes,
                                                            unsigned long long* __restrict__ offsets, uint32_t n, uint8_t* __restrict__ dst, size_t dst_cap,
                                                            const unsigned long long* __restrict__ src_offsets)
{
    const uint32_t f = blockIdx.y;
    const uint32_t nvec = (sizes[f] + 15u) / 16u;
    const unsigned long long o = offsets[f];
    const unsigned long long so = src_offsets ? src_offsets[f] : (unsigned long long)f * stride;
    if (o + (unsigned long long)nvec * 16ull > dst_cap || (so & 15ull)) {
        // the file does not fit (or its source is not 16-byte aligned): it is NOT copied, and bit 63 of offsets[n] (the total)
        // tells the caller so
        if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(&offsets[n], 1ull << 63);
        return;
    }
    const uint4* src = reinterpret_cast<const uint4*>(files + so);
    uint4* d = reinterpret_cast<uint4*>(dst + o);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += gridDim.x * blockDim.x) d[i] = src[i];
}

void launch_compact(const uint8_t* files, size_t stride, const uint32_t* sizes, uint32_t n, uint8_t* dst, size_t dst_cap,
                    unsigned long long* offsets, cudaStream_t s, const unsigned long long* src_offsets)
{
    compact_offsets_kernel<<<1, 1024, 0, s>>>(sizes, n, offsets);
    dim3 grid(64, n);
    compact_copy_kernel<<<grid, 256, 0, s>>>(files, stride, sizes, offsets, n, dst, dst_cap, src_offsets);
}

}  // namespace fpngb
