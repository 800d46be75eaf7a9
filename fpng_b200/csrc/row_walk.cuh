// fpng_b200/csrc/row_walk.cuh -- warp-level helpers shared by the encode, PNG encode and decode kernels: byte-wise filter
// arithmetic, the row carry of the scanline walker (row_walk16.cuh), warp sums and scans, and the stored-block row copy.
#pragma once
#include "common.cuh"

namespace fpngb {

constexpr uint32_t kFullMask = 0xFFFFFFFFu;

__device__ __forceinline__ uint32_t vsub4(uint32_t a, uint32_t b)
{
    // per-byte a - b (mod 256) without inter-byte borrows
    uint32_t d = (a | 0x80808080u) - (b & 0x7F7F7F7Fu);
    return d ^ ((a ^ ~b) & 0x80808080u);
}

__device__ __forceinline__ uint32_t ld_u8(const uint8_t* p) { return __ldg(p); }

// Warp-uniform state carried from one warp step of a scanline to the next.
struct RowCarry {
    uint32_t prev_px;   // filtered value of the pixel left of this step (lane 31's last pixel)
    uint32_t run;       // pixels of the pending, unfinished match token (0..M-1)
};

__device__ __forceinline__ uint32_t warp_sum_u32(uint32_t v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFullMask, v, o);
    return v;
}
__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFullMask, v, o);
    return v;
}
__device__ __forceinline__ uint32_t warp_excl_scan_u32(uint32_t v, uint32_t lane, uint32_t& total)
{
    uint32_t s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t n = __shfl_up_sync(kFullMask, s, o);
        if (lane >= (uint32_t)o) s += n;
    }
    total = __shfl_sync(kFullMask, s, 31);
    return s - v;
}

// exclusive prefix of v over the block (blockDim.x a multiple of 32, s_warp one entry per warp); total: the block sum
__device__ __forceinline__ unsigned long long block_excl_scan_u64(unsigned long long v, unsigned long long* s_warp, unsigned long long& total)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    unsigned long long s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long n = __shfl_up_sync(kFullMask, s, o);
        if (lane >= (uint32_t)o) s += n;
    }
    if (lane == 31) s_warp[warp] = s;
    __syncthreads();
    unsigned long long base = 0, tot = 0;
    for (uint32_t i = 0; i < nwarps; i++) { const unsigned long long x = s_warp[i]; if (i < warp) base += x; tot += x; }
    __syncthreads();
    total = tot;
    return base + s - v;
}

// Source bytes of a stored row, in PNG byte order: byte i of an interleaved scanline, or of a planar one (channel i % CHANS
// of pixel i / CHANS, planes chan_stride bytes apart)
struct RowBytes {
    const uint8_t* p;
    __device__ __forceinline__ uint32_t operator()(unsigned long long i) const { return ld_u8(p + i); }
};
template <int CHANS>
struct PlaneBytes {
    const uint8_t* p; size_t chan_stride;
    __device__ __forceinline__ uint32_t operator()(unsigned long long i) const
    {
        const unsigned long long x = i / CHANS;
        return ld_u8(p + x + (i - x * CHANS) * chan_stride);
    }
};

// Stored-block fallback for one row (fpng.cpp:818-866): stream byte s (row y, column t; t == 0 is the filter byte 0)
// lands at zlib offset 2 + 5 * (s / 65535 + 1) + s.  The row is copied block segment by block segment with 32-bit stores
// (source words rebuilt from byte loads that hit L1); also produces the row's Adler partials over the raw bytes.
template <class Src>
__device__ __forceinline__ void store_row_raw(const Src& at, uint8_t* __restrict__ zl, uint32_t y, uint32_t bpl, uint32_t lane, uint2* adler_out)
{
    const unsigned long long n = (unsigned long long)bpl + 1ull;
    const unsigned long long s0 = (unsigned long long)y * n;
    unsigned long long A = 0, B = 0;                      // sum v, sum t*v  (t = index inside the row's stream)
    unsigned long long t = 0;                              // next stream index of the row to copy
    while (t < n) {
        const unsigned long long s = s0 + t, blk = s / 65535ull;
        const unsigned long long seg = min(n - t, (blk + 1ull) * 65535ull - s);      // bytes until the row or the block ends
        uint8_t* dst = zl + 2ull + 5ull * (blk + 1ull) + s;
        // source of stream index t is 0 (filter) for t == 0, row byte t-1 otherwise
        unsigned long long done = 0;
        if (t == 0) { if (lane == 0) dst[0] = 0; done = 1; }
        const unsigned long long src = t + done - 1ull;
        uint8_t* d = dst + done;
        const unsigned long long len = seg - done;
        const uint32_t head = (uint32_t)min((unsigned long long)((4u - ((uintptr_t)d & 3u)) & 3u), len);
        if (lane < head) { const uint32_t v = at(src + lane); d[lane] = (uint8_t)v; A += v; B += (t + done + lane) * v; }
        const unsigned long long body = (len - head) >> 2;
        const unsigned long long sb = src + head; uint8_t* db = d + head;
        const unsigned long long tb = t + done + head;
        for (unsigned long long j = lane; j < body; j += 32) {
            const unsigned long long q = sb + 4ull * j;
            const uint32_t v = at(q) | (at(q + 1) << 8) | (at(q + 2) << 16) | (at(q + 3) << 24);
            *reinterpret_cast<uint32_t*>(db + 4ull * j) = v;
            const uint32_t t1 = __dp4a(v, 0x01010101u, 0u), t2 = __dp4a(v, 0x03020100u, 0u);
            A += t1; B += (tb + 4ull * j) * t1 + t2;
        }
        const uint32_t tail = (uint32_t)((len - head) & 3ull);
        if (lane < tail) { const unsigned long long o = head + 4ull * body + lane; const uint32_t v = at(src + o); d[o] = (uint8_t)v; A += v; B += (t + done + o) * v; }
        t += seg;
    }
    A = warp_sum_u64(A); B = warp_sum_u64(B);
    if (lane == 0) *adler_out = make_uint2((uint32_t)(A % kAdlerMod), (uint32_t)((n * A - B) % kAdlerMod));
}
__device__ __forceinline__ void store_row_raw(const uint8_t* __restrict__ cur, uint8_t* __restrict__ zl, uint32_t y, uint32_t bpl,
                                              uint32_t lane, uint2* adler_out)
{
    store_row_raw(RowBytes{cur}, zl, y, bpl, lane, adler_out);
}

}  // namespace fpngb
