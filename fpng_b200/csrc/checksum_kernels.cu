// fpng_b200/csrc/checksum_kernels.cu -- checksums of flat buffers and compaction of encoded batches.
//
// host_crc32: the byte-table CRC-32 of short host buffers (chunk headers, IHDR, fpngb_crc32 below 4 KiB or before fpngb_init);
// longer buffers go through idat_crc_stream_kernel (crc_stream_kernel.cu).  adler_buffer_kernel: the Adler-32 partials of
// fpngb_adler32.  compact_*_kernel: one contiguous buffer from a batch of encoded files.
#include "kernels.cuh"
#include "crc_math.cuh"

namespace fpngb {

uint32_t host_crc32(const void* data, size_t n, uint32_t prev)
{
    static constexpr CrcByteTable t = crc_byte_table();
    const uint8_t* p = (const uint8_t*)data;
    uint32_t c = ~prev;
    for (size_t i = 0; i < n; i++) c = t.t[(c ^ p[i]) & 0xFF] ^ (c >> 8);
    return ~c;
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
