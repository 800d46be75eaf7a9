// fpng_b200/csrc/row_walk.cuh -- warp-per-scanline tokeniser shared by the scan, histogram and pack kernels.
//
// One warp owns one scanline.  It walks the row in steps of 128 pixels; lane l owns the 4 consecutive
// pixels [128*step + 4*l, +4).  For every step the warp
//   1. loads the current and the previous scanline (PNG filter 2 "Up", filter 0 on row 0:
//      fpng.cpp:1592-1660, 1696) and forms the filtered pixels d = cur - prev (byte-wise, mod 256);
//   2. classifies every pixel as literal / covered-by-RLE-match exactly like the reference's greedy
//      scalar loop (fpng.cpp:1182-1243 RGB, 1468-1558 RGBA; 2-pass: 1021-1084, 1299-1363), using the
//      data-parallel restatement of SURVEY.md Appendix B: a run of pixels equal to their left neighbour
//      is cut into match tokens of M = 85 (RGB) / 63 (RGBA) pixels from the run start, and each token
//      is attributed to the pixel where it ENDS (full token) or to the literal that follows it /
//      the end of the row (remainder token), which preserves the token order of the serial coder.
//
// The run phase entering a lane comes from one ballot + one shuffle; everything else is lane-local.
#pragma once
#include "common.cuh"

namespace fpngb {

constexpr uint32_t kFullMask = 0xFFFFFFFFu;
constexpr int kPixPerLane = 4;
constexpr int kPixPerStep = 128;

enum LoadMode : int {
    kLoadBytes = 0,   // any alignment: byte loads
    kLoadWords = 1,   // every scanline starts 4-byte aligned and bpl % 4 == 0 (RGB additionally w % 4 == 0)
    kLoadVec16 = 2    // RGBA only: every scanline starts 16-byte aligned and w % 4 == 0
};

__device__ __forceinline__ uint32_t vsub4(uint32_t a, uint32_t b)
{
    // per-byte a - b (mod 256) without inter-byte borrows
    uint32_t d = (a | 0x80808080u) - (b & 0x7F7F7F7Fu);
    return d ^ ((a ^ ~b) & 0x80808080u);
}

__device__ __forceinline__ uint32_t ld_u8(const uint8_t* p) { return __ldg(p); }

// Load the lane's 4 pixels (4*CHANS bytes at byte offset `bo` of a scanline) as CHANS little-endian
// words in memory order; bytes at or beyond `bpl` read as zero.
template <int CHANS, int MODE>
__device__ __forceinline__ void load_lane_words(const uint8_t* __restrict__ row, uint32_t bo, uint32_t bpl, uint32_t (&wd)[CHANS])
{
    if (MODE == kLoadVec16 && CHANS == 4) {
        if (bo < bpl) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(row + bo));
            wd[0] = v.x; wd[1] = v.y; wd[2] = v.z; wd[CHANS - 1] = v.w;
        } else {
#pragma unroll
            for (int i = 0; i < CHANS; i++) wd[i] = 0;
        }
    } else if (MODE == kLoadWords) {
#pragma unroll
        for (int i = 0; i < CHANS; i++)
            wd[i] = (bo + 4u * i < bpl) ? __ldg(reinterpret_cast<const uint32_t*>(row + bo) + i) : 0u;
    } else {
#pragma unroll
        for (int i = 0; i < CHANS; i++) {
            uint32_t v = 0;
#pragma unroll
            for (int b = 0; b < 4; b++) {
                const uint32_t o = bo + 4u * i + b;
                if (o < bpl) v |= ld_u8(row + o) << (8 * b);
            }
            wd[i] = v;
        }
    }
}

template <int CHANS>
__device__ __forceinline__ void words_to_pixels(const uint32_t (&wd)[CHANS], uint32_t (&px)[4])
{
    if (CHANS == 4) {
#pragma unroll
        for (int k = 0; k < 4; k++) px[k] = wd[k];
    } else {
        px[0] = wd[0] & 0x00FFFFFFu;
        px[1] = __byte_perm(wd[0], wd[1], 0x4543) & 0x00FFFFFFu;   // bytes 3,4,5
        px[2] = __byte_perm(wd[1], wd[2], 0x4432) & 0x00FFFFFFu;   // bytes 6,7,8  (wd[1] bytes 2,3 ; wd[2] byte 0)
        px[3] = wd[2] >> 8;                                         // bytes 9,10,11
    }
}

// Warp-uniform state carried from one 128-pixel step to the next.
struct RowCarry {
    uint32_t prev_px;   // filtered value of the pixel left of this step (lane 31's last pixel)
    uint32_t run;       // pixels of the pending, unfinished match token (0..M-1)
};

// What the lane has to emit for its 4 pixel slots in this step, in order:
//   for k in 0..3:  [match of mlen[k] pixels, if mlen[k] != 0]  [literal px[k], if litmask bit k]
//   then            [match of tail pixels, if tail != 0]   (only on the lane that holds the row's last pixel)
struct LaneTokens {
    uint32_t px[4];
    uint32_t mlen[4];
    uint32_t tail;
    uint32_t litmask;
    uint32_t nvp;       // valid pixels in this lane (0..4)
    uint32_t left;      // filtered pixel left of px[0] (the previous lane's / step's last pixel)
};

// Pixel value of the run that a pending match flushed at slot k (mlen[k], k = 0..3) or at the row end (k = nvp) covers:
// the run's last pixel sits right before slot k.
__device__ __forceinline__ uint32_t run_pixel_before(const LaneTokens& t, uint32_t k)
{
    return k == 0 ? t.left : (k == 1 ? t.px[0] : (k == 2 ? t.px[1] : (k == 3 ? t.px[2] : t.px[3])));
}

template <int CHANS>
__device__ __forceinline__ void classify_step(LaneTokens& t, uint32_t p0, uint32_t w, RowCarry& carry, uint32_t lane)
{
    constexpr uint32_t M = max_match_pixels(CHANS);
    const uint32_t nvp = t.nvp;
    uint32_t left = __shfl_up_sync(kFullMask, t.px[3], 1);
    if (lane == 0) left = carry.prev_px;
    t.left = left;

    uint32_t eqmask = 0;
    if (nvp > 0 && p0 > 0 && t.px[0] == left) eqmask |= 1u;
#pragma unroll
    for (int k = 1; k < 4; k++)
        if ((uint32_t)k < nvp && t.px[k] == t.px[k - 1]) eqmask |= 1u << k;
    const uint32_t validmask = (1u << nvp) - 1u;
    const uint32_t litmask = validmask & ~eqmask;
    t.litmask = litmask;

    // equal pixels trailing the lane's last literal (or all of them when the lane has no literal)
    const uint32_t trail = litmask ? (nvp - 1u - (31u - (uint32_t)__clz((int)litmask))) : nvp;
    const uint32_t has_lit = __ballot_sync(kFullMask, litmask != 0);
    const uint32_t lower = has_lit & ((1u << lane) - 1u);
    const uint32_t src = lower ? (31u - (uint32_t)__clz((int)lower)) : 0u;
    const uint32_t src_trail = __shfl_sync(kFullMask, trail, src);
    uint32_t run = lower ? (src_trail + 4u * (lane - src - 1u)) : (carry.run + 4u * lane);
    run %= M;

#pragma unroll
    for (int k = 0; k < 4; k++) {
        t.mlen[k] = 0;
        if ((uint32_t)k < nvp) {
            if (eqmask & (1u << k)) {
                if (++run == M) { t.mlen[k] = M; run = 0; }
            } else {
                t.mlen[k] = run; run = 0;
            }
        }
    }
    t.tail = (nvp > 0 && p0 + nvp == w) ? run : 0u;

    carry.prev_px = __shfl_sync(kFullMask, t.px[3], 31);
    carry.run = __shfl_sync(kFullMask, run, 31);
}

// Loads one step of a scanline, applies the Up filter, returns the filtered words (memory order, zero
// beyond the row) and the lane's pixels.
template <int CHANS, int MODE>
__device__ __forceinline__ void load_filtered_step(const uint8_t* __restrict__ cur, const uint8_t* __restrict__ prev /*null on row 0*/,
                                                   uint32_t bo, uint32_t bpl, uint32_t (&dw)[CHANS], uint32_t (&px)[4])
{
    uint32_t cw[CHANS];
    load_lane_words<CHANS, MODE>(cur, bo, bpl, cw);
    if (prev) {
        uint32_t pw[CHANS];
        load_lane_words<CHANS, MODE>(prev, bo, bpl, pw);
#pragma unroll
        for (int i = 0; i < CHANS; i++) dw[i] = vsub4(cw[i], pw[i]);
    } else {
#pragma unroll
        for (int i = 0; i < CHANS; i++) dw[i] = cw[i];
    }
    words_to_pixels<CHANS>(dw, px);
}

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
