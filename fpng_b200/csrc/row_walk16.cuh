// fpng_b200/csrc/row_walk16.cuh -- the encoder's scanline walker: 16 consecutive pixels per lane, 512 per warp step.
//
// The tokenisation of the reference's greedy scalar coder (fpng.cpp:1182-1243 RGB, 1468-1558 RGBA; 2-pass: 1021-1084,
// 1299-1363) restated data-parallel (SURVEY.md Appendix B): a run of pixels equal to their left neighbour is cut into match
// tokens of M = 85 (RGB) / 63 (RGBA) pixels from the run start, and each token is attributed to the pixel where it ENDS (full
// token) or to the literal that follows it / the end of the row (remainder token), which preserves the serial token order.
// Per warp step:
//   1. one elected lane issues a TMA bulk copy (cp.async.bulk + mbarrier) of the step's 512 cur and prev pixels into the
//      warp's shared-memory tile, one step ahead of the computation;
//   2. each lane reads its own 16 consecutive pixels with 128-bit shared loads, subtracts the previous scanline (PNG
//      filter 2 "Up", fpng.cpp:1605-1652) and accumulates the Adler-32 partial sums;
//   3. equality with the left pixel gives a 16-bit mask per lane; the run phase entering the lane is one ballot + one
//      shuffle; the lane then walks its pixels.
// The staged loaders require every scanline to start 16-byte aligned and bpl % 16 == 0 (RGBA: w % 4 == 0, RGB: w % 16 == 0);
// the direct and planar loaders below take any other shape.
#pragma once
#include "row_walk.cuh"

namespace fpngb {

constexpr int kPix16 = 16;                       // pixels per lane per step
constexpr int kStep16 = 32 * kPix16;             // pixels per warp step
// ---- TMA (bulk async copy) staging ------------------------------------------------------------------------------
// One elected lane per warp issues ONE `cp.async.bulk` per scanline per step (cur and prev: 512 pixels = 1536 / 2048
// contiguous bytes each) into the warp's shared-memory tile and arms the warp's mbarrier with the byte count; all lanes
// wait on the mbarrier phase, read their own 16 pixels (48 / 64 contiguous bytes per lane) into registers, and the next
// step's copies are issued while this step is processed.  SASS: UBLKCP + SYNCS.
constexpr int kTileLaneBytes = 80;                      // padded per-lane slot of the cp.async (RGBA) variant

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(void* mbar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" :: "r"(smem_u32(mbar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(void* mbar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" :: "r"(smem_u32(mbar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(void* mbar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" :: "r"(smem_u32(mbar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, void* mbar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n"
                 :: "r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(bytes), "r"(smem_u32(mbar)) : "memory");
}


// The encode kernels are bound by the ALU pipe (LOP3 / SHF / IADD3 / ISETP / SEL; ncu: ~77 % active) while the FMA pipe idles (~17 %).
// Multipliers the compiler cannot fold keep a few add / shift-add steps on the FMA pipe as IMAD with a constant-bank operand
// (a literal 2 or -1 would be strength-reduced to LEA / IADD3, ALU-pipe instructions): {2, -1, 2^8, 2^16, 2^24, 8}.
static __constant__ uint32_t c_fma_k[6] = {2u, 0xFFFFFFFFu, 1u << 8, 1u << 16, 1u << 24, 8u};

// Adler-32 partial sums of one 16-byte chunk at byte offset 16 * I of the lane's bytes: t1 += sum of bytes, t2 += sum of (position inside
// the lane's bytes) * byte.  The position weights fold the chunk offset (<= 63: a u8), so a step needs ONE 64-bit multiply-add per lane
// (lane_base * T1 + T2) instead of one per chunk.
template <int I>
__device__ __forceinline__ void adler_chunk16(const uint4& d, uint32_t& t1, uint32_t& t2)
{
    constexpr uint32_t kW = 0x03020100u + 0x01010101u * (16u * I);
    t1 = __dp4a(d.x, 0x01010101u, t1); t2 = __dp4a(d.x, kW, t2);
    t1 = __dp4a(d.y, 0x01010101u, t1); t2 = __dp4a(d.y, kW + 0x04040404u, t2);
    t1 = __dp4a(d.z, 0x01010101u, t1); t2 = __dp4a(d.z, kW + 0x08080808u, t2);
    t1 = __dp4a(d.w, 0x01010101u, t1); t2 = __dp4a(d.w, kW + 0x0C0C0C0Cu, t2);
}
template <int I, int N> struct AdlerChunks {
    __device__ __forceinline__ static void run(const uint32_t* dw, uint32_t& t1, uint32_t& t2)
    {
        adler_chunk16<I>(make_uint4(dw[4 * I], dw[4 * I + 1], dw[4 * I + 2], dw[4 * I + 3]), t1, t2);
        AdlerChunks<I + 1, N>::run(dw, t1, t2);
    }
};
template <int N> struct AdlerChunks<N, N> { __device__ __forceinline__ static void run(const uint32_t*, uint32_t&, uint32_t&) {} };
// all CHANS chunks of a lane's filtered words; sumA / sumB are the scanline's running sums (bytes, position-weighted bytes)
template <int CHANS>
__device__ __forceinline__ void adler_lane16(const uint32_t (&dw)[4 * CHANS], uint32_t lane_base, uint32_t& sumA, unsigned long long& sumB)
{
    uint32_t t1 = 0, t2 = 0;
    AdlerChunks<0, CHANS>::run(dw, t1, t2);
    sumA += t1;
    sumB += (unsigned long long)lane_base * t1 + t2;
}

template <int CHANS>
struct Walk16Tma {
    static constexpr int kWords = 4 * CHANS;     // filtered words per lane per step (16 pixels)
    static constexpr uint32_t kStepBytes = kStep16 * CHANS;
    static constexpr uint32_t kTile = kStepBytes;             // one scanline step: 1536 (RGB) / 2048 (RGBA) bytes
    static constexpr uint32_t kMbarOfs = 2 * kTile;           // the warp's mbarrier sits behind the cur and prev tiles
    static constexpr int kWarpBytes = 2 * kTile + 16;         // shared memory per warp

    __device__ __forceinline__ void init(uint32_t lane, uint8_t* warp_tiles)
    {
        if (lane == 0) mbar_init(warp_tiles + kMbarOfs, 1);
        __syncwarp();
    }
    __device__ __forceinline__ void bind(const uint8_t*, const uint8_t*) {}

    // issue the bulk copies of one step (lane 0 only) into this warp's tile
    __device__ __forceinline__ void prefetch(const uint8_t* __restrict__ cur, const uint8_t* __restrict__ prev, uint32_t step, uint32_t bpl,
                                             uint32_t lane, uint8_t* warp_tiles) const
    {
        if (lane == 0) {
            const uint32_t b = step * kStepBytes;
            const uint32_t bytes = min(kStepBytes, bpl - b);              // bpl % 16 == 0
            void* mbar = warp_tiles + kMbarOfs;
            // order the previous step's generic-proxy reads of the tile before the async-proxy writes
            asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
            mbar_expect_tx(mbar, prev ? 2u * bytes : bytes);
            tma_bulk_g2s(warp_tiles, cur + b, bytes, mbar);
            if (prev) tma_bulk_g2s(warp_tiles + kTile, prev + b, bytes, mbar);
        }
    }

    // wait for the step to land, read the lane's 16 pixels, apply the Up filter (fpng.cpp:1605-1652), optionally add the
    // Adler partials (sum of bytes, position-weighted sum) of these 16*CHANS bytes
    // `phase` counts the prefetches consumed so far by this warp (mbarrier parity); `step` is the position inside the row
    template <bool kAdler>
    __device__ __forceinline__ void consume(bool have_prev, uint32_t phase, uint32_t step, uint32_t bpl, uint32_t lane, uint8_t* warp_tiles,
                                            uint32_t (&dw)[kWords], uint32_t& sumA, unsigned long long& sumB) const
    {
        mbar_wait(warp_tiles + kMbarOfs, phase & 1u);
        const uint8_t* tc = warp_tiles + lane * (16 * CHANS);
        const uint8_t* tp = tc + kTile;
        const uint32_t lane_base = step * kStepBytes + lane * (16u * CHANS);     // byte offset of the lane's first byte in the row
        if ((step + 1u) * kStepBytes <= bpl) {                                   // warp-uniform: the whole step lies inside the scanline
#pragma unroll
            for (int i = 0; i < CHANS; i++) {
                uint4 d = *reinterpret_cast<const uint4*>(tc + i * 16);
                if (have_prev) {
                    const uint4 q = *reinterpret_cast<const uint4*>(tp + i * 16);
                    d.x = vsub4(d.x, q.x); d.y = vsub4(d.y, q.y); d.z = vsub4(d.z, q.z); d.w = vsub4(d.w, q.w);
                }
                dw[4 * i] = d.x; dw[4 * i + 1] = d.y; dw[4 * i + 2] = d.z; dw[4 * i + 3] = d.w;
            }
        } else {
#pragma unroll
            for (int i = 0; i < CHANS; i++) {
                uint4 d = make_uint4(0, 0, 0, 0);
                if (lane_base + 16u * i < bpl) {                                 // bytes beyond the scanline were not copied
                    d = *reinterpret_cast<const uint4*>(tc + i * 16);
                    if (have_prev) {
                        const uint4 q = *reinterpret_cast<const uint4*>(tp + i * 16);
                        d.x = vsub4(d.x, q.x); d.y = vsub4(d.y, q.y); d.z = vsub4(d.z, q.z); d.w = vsub4(d.w, q.w);
                    }
                }
                dw[4 * i] = d.x; dw[4 * i + 1] = d.y; dw[4 * i + 2] = d.z; dw[4 * i + 3] = d.w;
            }
        }
        if (kAdler) adler_lane16<CHANS>(dw, lane_base, sumA, sumB);
        __syncwarp();                                                            // every lane has its pixels: the tile may be refilled
    }

    __device__ __forceinline__ static void pixels(const uint32_t (&dw)[kWords], uint32_t (&px)[16])
    {
        if (CHANS == 4) {
#pragma unroll
            for (int k = 0; k < 16; k++) px[k] = dw[k];
        } else {
#pragma unroll
            for (int g = 0; g < 4; g++) {
                const uint32_t w0 = dw[3 * g], w1 = dw[3 * g + 1], w2 = dw[3 * g + 2];
                px[4 * g] = w0 & 0x00FFFFFFu;
                px[4 * g + 1] = __byte_perm(w0, w1, 0x4543) & 0x00FFFFFFu;
                px[4 * g + 2] = __byte_perm(w1, w2, 0x4432) & 0x00FFFFFFu;
                px[4 * g + 3] = w2 >> 8;
            }
        }
    }
};

// ---- cp.async (LDGSTS) staging into padded slots ------------------------------------------------------------------
// RGBA variant: 64 contiguous bytes per lane would make the 128-bit shared reads 4-way bank conflicted, and that costs
// more than it saves on the LSU-heavy RGBA kernels (measured: scan 1.71 ms with the linear TMA tile vs 1.48 ms padded).
// Lane l copies the 16-byte chunks #(j*32 + l) (coalesced in HBM) into the 80-byte padded slot of the lane that owns the
// pixels; same single-stage pipeline (consume into registers, then refill for the next step).
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src, bool valid)
{
    const int src_bytes = valid ? 16 : 0;                // 0 -> the 16 destination bytes are zero-filled, nothing is read
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" :: "r"(smem_u32(smem_dst)), "l"(gmem_src), "r"(src_bytes) : "memory");
}

template <int CHANS>
struct Walk16Padded {
    static constexpr int kWords = 4 * CHANS;
    static constexpr int kPadTile = 32 * kTileLaneBytes;
    static constexpr int kWarpBytes = 2 * kPadTile;           // shared memory per warp
    uint32_t soff[CHANS];                        // byte offsets inside a tile where this lane's copies land
    __device__ __forceinline__ void bind(const uint8_t*, const uint8_t*) {}

    __device__ __forceinline__ void init(uint32_t lane, uint8_t*)
    {
#pragma unroll
        for (int j = 0; j < CHANS; j++) {
            const uint32_t q = j * 32u + lane;   // chunk index inside the step
            soff[j] = (q / CHANS) * kTileLaneBytes + (q % CHANS) * 16u;
        }
    }
    __device__ __forceinline__ void prefetch(const uint8_t* __restrict__ cur, const uint8_t* __restrict__ prev, uint32_t step, uint32_t bpl,
                                             uint32_t lane, uint8_t* warp_tiles) const
    {
        const uint32_t step_base = step * (uint32_t)(kStep16 * CHANS);
#pragma unroll
        for (int j = 0; j < CHANS; j++) {
            const uint32_t b = step_base + (j * 32u + lane) * 16u;
            const bool valid = b < bpl;
            cp_async16(warp_tiles + soff[j], cur + (valid ? b : 0u), valid);
            if (prev) cp_async16(warp_tiles + kPadTile + soff[j], prev + (valid ? b : 0u), valid);
        }
        asm volatile("cp.async.commit_group;\n" ::: "memory");
    }
    template <bool kAdler>
    __device__ __forceinline__ void consume(bool have_prev, uint32_t, uint32_t step, uint32_t, uint32_t lane, uint8_t* warp_tiles,
                                            uint32_t (&dw)[kWords], uint32_t& sumA, unsigned long long& sumB) const
    {
        asm volatile("cp.async.wait_group 0;\n" ::: "memory");
        __syncwarp();
        const uint8_t* tc = warp_tiles + lane * kTileLaneBytes;
        const uint8_t* tp = tc + kPadTile;
        const uint32_t lane_base = (step * (uint32_t)kStep16 + lane * (uint32_t)kPix16) * CHANS;
#pragma unroll
        for (int i = 0; i < CHANS; i++) {
            uint4 d = *reinterpret_cast<const uint4*>(tc + i * 16);
            if (have_prev) {
                const uint4 q = *reinterpret_cast<const uint4*>(tp + i * 16);
                d.x = vsub4(d.x, q.x); d.y = vsub4(d.y, q.y); d.z = vsub4(d.z, q.z); d.w = vsub4(d.w, q.w);
            }
            dw[4 * i] = d.x; dw[4 * i + 1] = d.y; dw[4 * i + 2] = d.z; dw[4 * i + 3] = d.w;
        }
        if (kAdler) adler_lane16<CHANS>(dw, lane_base, sumA, sumB);
        __syncwarp();
    }
    __device__ __forceinline__ static void pixels(const uint32_t (&dw)[kWords], uint32_t (&px)[16])
    {
#pragma unroll
        for (int k = 0; k < 16; k++) px[k] = dw[k];
    }
};

// ---- direct loads for scanlines of ANY alignment / width --------------------------------------------------------------
// Real-world widths (687 x 3 = 2061-byte scanlines) give rows that start at arbitrary byte addresses, which neither TMA bulk
// copies nor cp.async (16-byte granules) can stage.  Here every lane loads the aligned 16-byte chunks that cover its own 16
// pixels (48 / 64 bytes: 4 or 5 LDG.128) and realigns them in registers with funnel shifts.  The lane stride is a multiple
// of 16 bytes, so the misalignment (address & 15) is the same for every lane of the warp: the word part of the shift is a
// warp-uniform switch, the byte part one SHF per word.  Bytes at or beyond the end of the scanline read as zero and chunks
// that lie completely outside the lane's byte range are not loaded (nothing is read beyond the 16-byte chunk that holds the
// scanline's last byte).
template <int CHANS>
struct Walk16Direct {
    static constexpr int kWords = 4 * CHANS;
    static constexpr int kWarpBytes = 0;                      // no staging buffer
    __device__ __forceinline__ void init(uint32_t, uint8_t*) {}
    __device__ __forceinline__ void prefetch(const uint8_t*, const uint8_t*, uint32_t, uint32_t, uint32_t, uint8_t*) const {}

    __device__ __forceinline__ static void load_lane(const uint8_t* __restrict__ ptr, uint32_t nbytes, uint32_t (&out)[kWords])
    {
        constexpr int kChunks = CHANS + 1;                    // 16-byte chunks that can overlap the lane's 16 * CHANS bytes
        const uint32_t delta = (uint32_t)((uintptr_t)ptr & 15u);
        const uint4* a = reinterpret_cast<const uint4*>(ptr - delta);
        uint32_t W[4 * kChunks + 1];
#pragma unroll
        for (int j = 0; j < kChunks; j++) {
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (16u * j < nbytes + delta) v = __ldg(a + j);
            W[4 * j] = v.x; W[4 * j + 1] = v.y; W[4 * j + 2] = v.z; W[4 * j + 3] = v.w;
        }
        W[4 * kChunks] = 0u;
        const uint32_t r = (delta & 3u) * 8u;
        switch (delta >> 2) {                                 // warp-uniform
        case 0:
#pragma unroll
            for (int i = 0; i < kWords; i++) out[i] = __funnelshift_r(W[i], W[i + 1], r);
            break;
        case 1:
#pragma unroll
            for (int i = 0; i < kWords; i++) out[i] = __funnelshift_r(W[i + 1], W[i + 2], r);
            break;
        case 2:
#pragma unroll
            for (int i = 0; i < kWords; i++) out[i] = __funnelshift_r(W[i + 2], W[i + 3], r);
            break;
        default:
#pragma unroll
            for (int i = 0; i < kWords; i++) out[i] = __funnelshift_r(W[i + 3], W[i + 4], r);
            break;
        }
        if (nbytes < 16u * CHANS) {                           // the lane that holds the end of the scanline: zero the bytes beyond it
#pragma unroll
            for (int i = 0; i < kWords; i++) {
                const uint32_t have = nbytes > 4u * i ? nbytes - 4u * i : 0u;
                out[i] = have >= 4u ? out[i] : (have ? (out[i] & ((1u << (8u * have)) - 1u)) : 0u);
            }
        }
    }

    template <bool kAdler>
    __device__ __forceinline__ void consume(bool have_prev, uint32_t, uint32_t step, uint32_t bpl, uint32_t lane, uint8_t*,
                                            uint32_t (&dw)[kWords], uint32_t& sumA, unsigned long long& sumB) const
    {
        // cur / prev are passed through the object (the staging variants get them in prefetch)
        const uint32_t lane_base = (step * (uint32_t)kStep16 + lane * (uint32_t)kPix16) * CHANS;
        const uint32_t nbytes = lane_base < bpl ? min(16u * CHANS, bpl - lane_base) : 0u;
        if (nbytes) {
            load_lane(cur_ + lane_base, nbytes, dw);
            if (have_prev) {
                uint32_t pw[kWords];
                load_lane(prev_ + lane_base, nbytes, pw);
#pragma unroll
                for (int i = 0; i < kWords; i++) dw[i] = vsub4(dw[i], pw[i]);
                if (nbytes < 16u * CHANS) {                   // vsub4 of zero padding stays zero, nothing to fix
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < kWords; i++) dw[i] = 0u;
        }
        if (kAdler) adler_lane16<CHANS>(dw, lane_base, sumA, sumB);
    }
    __device__ __forceinline__ static void pixels(const uint32_t (&dw)[kWords], uint32_t (&px)[16]) { Walk16Tma<CHANS>::pixels(dw, px); }
    __device__ __forceinline__ void bind(const uint8_t* cur, const uint8_t* prev) { cur_ = cur; prev_ = prev; }
    const uint8_t* cur_ = nullptr; const uint8_t* prev_ = nullptr;
};

// ---- planar (CHW-style) scanlines: one byte plane per channel -------------------------------------------------------
// Byte (x, c) of a scanline is at cur + x + c * chan_stride.  Each lane loads its 16 bytes of every plane (cur and prev row)
// with Walk16Direct's realigning 128-bit loads (the lane stride is 16 bytes, so each plane's misalignment is warp-uniform),
// applies the Up filter per plane (vsub4 is byte-wise: filtering before interleaving is exact) and interleaves the planes
// with byte permutes into exactly the words the interleaved loaders deliver.  Pixels beyond the scanline read as zero.
template <int CHANS>
struct Walk16Planar {
    static constexpr int kWords = 4 * CHANS;
    static constexpr int kWarpBytes = 0;                      // no staging buffer
    __device__ __forceinline__ void init(uint32_t, uint8_t*) {}
    __device__ __forceinline__ void prefetch(const uint8_t*, const uint8_t*, uint32_t, uint32_t, uint32_t, uint8_t*) const {}

    template <bool kAdler>
    __device__ __forceinline__ void consume(bool have_prev, uint32_t, uint32_t step, uint32_t bpl, uint32_t lane, uint8_t*,
                                            uint32_t (&dw)[kWords], uint32_t& sumA, unsigned long long& sumB) const
    {
        const uint32_t w = bpl / CHANS;
        const uint32_t p0 = step * (uint32_t)kStep16 + lane * (uint32_t)kPix16;
        const uint32_t np = p0 < w ? min(16u, w - p0) : 0u;
        uint32_t pl[CHANS][4];                               // 16 filtered bytes of each plane
        if (np) {
#pragma unroll
            for (int c = 0; c < CHANS; c++) {
                Walk16Direct<1>::load_lane(cur_ + p0 + c * cs_, np, pl[c]);
                if (have_prev) {
                    uint32_t q[4];
                    Walk16Direct<1>::load_lane(prev_ + p0 + c * cs_, np, q);
#pragma unroll
                    for (int i = 0; i < 4; i++) pl[c][i] = vsub4(pl[c][i], q[i]);
                }
            }
        } else {
#pragma unroll
            for (int c = 0; c < CHANS; c++)
#pragma unroll
                for (int i = 0; i < 4; i++) pl[c][i] = 0u;
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {                        // pixels 4j .. 4j+3
            const uint32_t r = pl[0][j], g = pl[1][j], b = pl[2][j];
            const uint32_t rg_lo = __byte_perm(r, g, 0x5140), rg_hi = __byte_perm(r, g, 0x7362);   // r0 g0 r1 g1 / r2 g2 r3 g3
            if (CHANS == 4) {
                const uint32_t a = pl[CHANS - 1][j];
                const uint32_t ba_lo = __byte_perm(b, a, 0x5140), ba_hi = __byte_perm(b, a, 0x7362);
                dw[4 * j] = __byte_perm(rg_lo, ba_lo, 0x5410);     dw[4 * j + 1] = __byte_perm(rg_lo, ba_lo, 0x7632);
                dw[4 * j + 2] = __byte_perm(rg_hi, ba_hi, 0x5410); dw[4 * j + 3] = __byte_perm(rg_hi, ba_hi, 0x7632);
            } else {
                dw[3 * j] = __byte_perm(rg_lo, b, 0x2410);                                    // r0 g0 b0 r1
                dw[3 * j + 1] = __byte_perm(__byte_perm(rg_lo, b, 0x0053), rg_hi, 0x5410);    // g1 b1 r2 g2
                dw[3 * j + 2] = __byte_perm(rg_hi, b, 0x7326);                                // b2 r3 g3 b3
            }
        }
        if (kAdler) adler_lane16<CHANS>(dw, p0 * CHANS, sumA, sumB);
    }
    __device__ __forceinline__ static void pixels(const uint32_t (&dw)[kWords], uint32_t (&px)[16]) { Walk16Tma<CHANS>::pixels(dw, px); }
    __device__ __forceinline__ void bind(const uint8_t* cur, const uint8_t* prev) { cur_ = cur; prev_ = prev; }
    __device__ __forceinline__ void planes(size_t chan_stride) { cs_ = chan_stride; }
    const uint8_t* cur_ = nullptr; const uint8_t* prev_ = nullptr; size_t cs_ = 0;
};

// RGB: linear TMA tile (48-byte lane stride is bank-conflict free for 128-bit reads); RGBA: padded cp.async tile.
template <int CHANS> struct Walk16Select { using type = Walk16Tma<CHANS>; };
template <> struct Walk16Select<4> { using type = Walk16Padded<4>; };
template <int CHANS> using Walk16 = typename Walk16Select<CHANS>::type;

struct Lane16 {
    uint32_t eqm;      // bit k: pixel k equals its left neighbour (valid pixels only)
    uint32_t litm;     // bit k: pixel k is a literal
    uint32_t nvp;      // valid pixels in this lane (0..16)
    uint32_t run;      // pending (unfinished) match length entering the lane, 0..M-1
    bool last;         // this lane holds the scanline's last pixel
};

// what the scan kernel hands to the pack kernel per lane and step: eqm | run << 16 | nvp << 23 | last << 28
__device__ __forceinline__ uint32_t lane_info16(const Lane16& t) { return t.eqm | (t.run << 16) | (t.nvp << 23) | (t.last ? (1u << 28) : 0u); }

// min(v, 1) as one VIMNMX (written in C++ the compiler turns it into compare + select: two ALU-pipe instructions)
__device__ __forceinline__ uint32_t nonzero01(uint32_t v) { uint32_t r; asm("min.u32 %0, %1, 1;\n" : "=r"(r) : "r"(v)); return r; }

template <int CHANS>
__device__ __forceinline__ Lane16 classify16(const uint32_t (&px)[16], uint32_t p0, uint32_t w, RowCarry& carry, uint32_t lane)
{
    constexpr uint32_t M = max_match_pixels(CHANS);
    Lane16 t;
    t.nvp = p0 < w ? min(16u, w - p0) : 0u;
    uint32_t left = __shfl_up_sync(kFullMask, px[15], 1);
    if (lane == 0) left = carry.prev_px;
    // bit k of `ne`: pixel k differs from its left neighbour.  Per pixel one ALU-pipe instruction (min) and two IMADs (difference,
    // shift-add into the mask) instead of compare + select + OR (see c_fma_k)
    const uint32_t kTwo = c_fma_k[0], kM1 = c_fma_k[1];
    uint32_t ne = 0;
#pragma unroll
    for (int k = 15; k >= 1; k--) ne = ne * kTwo + nonzero01(px[k - 1] * kM1 + px[k]);
    ne = ne * kTwo + (p0 > 0 ? nonzero01(left * kM1 + px[0]) : 1u);
    const uint32_t eq = ~ne;
    const uint32_t valid = (1u << t.nvp) - 1u;
    t.eqm = eq & valid;
    t.litm = valid & ~eq;
    t.last = t.nvp > 0 && p0 + t.nvp == w;

    const uint32_t trail = t.litm ? (t.nvp - 1u - (31u - (uint32_t)__clz((int)t.litm))) : t.nvp;
    const uint32_t has_lit = __ballot_sync(kFullMask, t.litm != 0);
    const uint32_t lower = has_lit & ((1u << lane) - 1u);
    const uint32_t src = lower ? (31u - (uint32_t)__clz((int)lower)) : 0u;
    const uint32_t src_trail = __shfl_sync(kFullMask, trail, src);
    const uint32_t run = lower ? (src_trail + 16u * (lane - src - 1u)) : (carry.run + 16u * lane);
    t.run = run % M;

    // carry for the next step: what lane 31 leaves pending
    const uint32_t out_run = t.litm ? trail : (t.run + t.nvp) % M;     // all-equal lane: phase advances by nvp
    carry.prev_px = __shfl_sync(kFullMask, px[15], 31);
    carry.run = __shfl_sync(kFullMask, out_run, 31);
    return t;
}

}  // namespace fpngb
