// fpng_b200/csrc/encode_fused.cu -- third-generation encoder: ONE pass over the pixels.
//
// The two-kernel encoder (encode16_kernels.cu) reads every pixel twice (scan: sizes only; pack: codes) because a scanline's
// position in the bit stream is only known after all earlier scanlines were sized.  This kernel reads the input ONCE:
//
//   * A CTA owns a "row group": R consecutive scanlines cut into S = ceil(w / 512) units of 512 pixels, one warp per unit
//     (R * S <= 8 warps).  Row groups are handed out in stream order by an atomic ticket, so a group only ever waits for
//     groups that are already running (decoupled look-back, no deadlock).
//   * Phase 1 (per warp): TMA / cp.async staged tile -> registers, Up filter (fpng.cpp:1592-1660), Adler partials
//     (fpng.cpp:403-487), pixel-equality mask.  The run phase entering a unit comes from the units to its left through
//     shared memory (a unit knows whether it holds a literal and how many equal pixels trail it).
//   * Phase 2 (per lane): the lane's 16 pixels are tokenised (fpng.cpp:1182-1243 / 1468-1558, SURVEY.md Appendix B) and their
//     Huffman codes appended to a LANE-LOCAL bit string in shared memory, starting at bit 0 -- no offsets are needed yet, the
//     code sizes fall out of the emission itself (this is what makes the separate sizing pass unnecessary).
//   * Phase 3: warp scan of the lane bit counts, CTA scan of the unit bit counts, then the group's bit count is published
//     and the look-back over earlier groups of the same image yields the group's position in the file.
//   * Phase 4: every lane copies its bit string to its place in the CTA's staging buffer (funnel shifts), the CTA writes the
//     staging words to the file shifted by the group's sub-word offset; the word a group shares with its successor travels
//     through the successor's descriptor ("tail"), so no atomics on the output and no pre-zeroed output are needed.
//
// A small finishing kernel (fused_finish_kernel) then applies the reference's compressed-vs-stored rule (fpng.cpp:567-588,
// 1705, 1728), writes the container header, the last partial word, IEND; Adler/CRC kernels run as before.  Images that fall
// back to stored blocks are rewritten by the stored path of the pack kernel.
#include "row_walk16.cuh"
#include "kernels.cuh"
#include "crc_math.cuh"
#include <string.h>

namespace fpngb {

// ---- CRC-32 of the IDAT chunk computed while the bits are still in shared memory (fpng.cpp:1797 does a second pass over the
// output with PCLMULQDQ folding, fpng.cpp:255-281).  The CRC is GF(2)-linear in the message BITS and Deflate packs bits
// LSB-first exactly like the reflected CRC consumes them, so a row group's bit string contributes
//        raw_crc(bit string, zero padded to whole words) * x^(bits between the padded end and the end of the message)
// independent of its (sub-byte) position.  The kernel stores the raw CRC per group; fused_crc_kernel multiplies the powers.
// Inside a group: lanes stride over the staging words (a register advanced over 32 words = 128 bytes per step: slice
// tables g_f128b), chunks of kCrcChunkWords words per warp, aligned to the END of the group's string so that the lane and
// chunk multipliers are constants (nibble tables in global memory, L1 resident).
constexpr uint32_t kCrcChunkWords = 256;          // words per warp chunk: 8 lane steps
__device__ uint32_t g_f128b[4][256];              // byte k of (reg ^ word) advanced over 128 bytes
__device__ uint32_t g_lane_mul[32][8][16];        // nibble tables: multiply by x^(32 * (32 - lane))
__device__ uint32_t g_chunk_mul[32][8][16];       // nibble tables: multiply by x^(32 * kCrcChunkWords * m)
__constant__ uint32_t c_fx_pow2[64];              // x^(2^k)

int fused_tables_init()
{
    static uint32_t f[4][256], lane[32][8][16], chunk[32][8][16], xp[64];
    crc_advance_tables(f, 128);
    for (uint32_t l = 0; l < 32; l++) crc_mul_table(lane[l], xpow(32ull * (32 - l)));
    for (uint32_t m = 0; m < 32; m++) crc_mul_table(chunk[m], xpow(32ull * kCrcChunkWords * m));
    crc_xpow2_table(xp);
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(g_f128b, f, sizeof f));
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(g_lane_mul, lane, sizeof lane));
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(g_chunk_mul, chunk, sizeof chunk));
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(c_fx_pow2, xp, sizeof xp));
    return 0;
}

constexpr int kFusedWarps = 8;                    // units per row group (upper bound)
constexpr uint32_t kStateAgg = 1ull, kStateIncl = 2ull;
constexpr unsigned long long kValueMask = (1ull << 62) - 1ull;
constexpr unsigned long long kTailReady = 1ull << 63;
constexpr uint32_t kSpinLimit = 1u << 22;         // a bug must fail the run, never hang the GPU

template <int CHANS> __host__ __device__ constexpr int fused_slot_words() { return CHANS == 3 ? 21 : 27; }   // lane-local bit string (odd: conflict-free)
template <int CHANS> __host__ __device__ constexpr int fused_unit_words() { return (512 * 12 * CHANS + 18 + 12 + 12) / 32 + 2; }   // staging words per unit, worst case
// scanline loader of the kernel: staged tiles (TMA / cp.async) for 16-byte aligned scanlines, direct realigning loads otherwise
template <int CHANS, bool DIRECT> struct FusedLoader { using type = Walk16<CHANS>; };
template <int CHANS> struct FusedLoader<CHANS, true> { using type = Walk16Direct<CHANS>; };
template <int CHANS, bool DIRECT> __host__ __device__ constexpr int fused_unit_bytes()
{
    using WK = typename FusedLoader<CHANS, DIRECT>::type;
    return WK::kWarpBytes > 32 * fused_slot_words<CHANS>() * 4 ? WK::kWarpBytes : 32 * fused_slot_words<CHANS>() * 4;
}

__device__ __forceinline__ void sts32(uint32_t saddr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;\n" :: "r"(saddr), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t lds32(uint32_t saddr) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];\n" : "=r"(v) : "r"(saddr) : "memory"); return v; }
__device__ __forceinline__ uint32_t lds32c(uint32_t saddr) { uint32_t v; asm("ld.shared.u32 %0, [%1];\n" : "=r"(v) : "r"(saddr)); return v; }   // tables: may be CSE'd
__device__ __forceinline__ void red_or32(uint32_t saddr, uint32_t v) { asm volatile("red.shared.or.b32 [%0], %1;\n" :: "r"(saddr), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long* p)
{
    unsigned long long v; asm volatile("ld.volatile.global.u64 %0, [%1];\n" : "=l"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void st_volatile_u64(unsigned long long* p, unsigned long long v)
{
    asm volatile("st.volatile.global.u64 [%0], %1;\n" :: "l"(p), "l"(v) : "memory");
}

// Lane-local bit string: the slot is private, so the word in progress can be stored on every put.  P is the running bit
// count; shifts use it modulo 32 (funnel shifts wrap), a put crosses into the next word iff bit 5 of P changes (len < 32).
struct LaneStager {
    uint32_t cur, P, dst;
    __device__ __forceinline__ void begin(uint32_t slot_saddr) { cur = 0u; P = 0u; dst = slot_saddr; }
    __device__ __forceinline__ void put(uint32_t code, uint32_t len)          // len < 32, code < 2^len
    {
        const uint32_t lo = cur | __funnelshift_l(0u, code, P);             // code << (P & 31)
        const uint32_t hi = __funnelshift_l(code, 0u, P);                    // bits spilling into the next word (0 when P & 31 == 0)
        const uint32_t P2 = P + len;
        sts32(dst, lo);
        if ((P ^ P2) & 32u) { dst += 4u; cur = hi; } else cur = lo;
        P = P2;
    }
    __device__ __forceinline__ uint32_t finish() { sts32(dst, cur); return P; }
};

#ifndef FPNGB_FUSED_TICKET
#define FPNGB_FUSED_TICKET 0
#endif
// fput_word*: literal table entries as (code, size) register pairs fetched with one 64-bit shared load, instead of one packed
// 32-bit word whose fields have to be shifted / masked apart (2 ALU instructions less per literal)
__device__ __forceinline__ uint2 lds64c(uint32_t saddr) { uint2 v; asm("ld.shared.v2.u32 {%0, %1}, [%2];\n" : "=r"(v.x), "=r"(v.y) : "r"(saddr)); return v; }
template <int POS>
__device__ __forceinline__ uint32_t flit_off8(uint32_t w, uint32_t nb)
{
    const uint32_t x = POS == 0 ? (w << 3) : (POS == 1 ? (w >> 5) : (POS == 2 ? (w >> 13) : (w >> 21)));
    return (x & 0x7F8u) | nb;
}
__device__ __forceinline__ void fput_pair2(LaneStager& bs, uint2 a, uint2 b) { bs.put(a.x | (b.x << a.y), a.y + b.y); }

__device__ __forceinline__ void fput_pair(LaneStager& bs, uint32_t a, uint32_t b)
{
    const uint32_t la = a >> 16;
    bs.put((a & 0xFFFFu) | ((b & 0xFFFFu) << la), la + (b >> 16));
}
__device__ __forceinline__ void fput_match(LaneStager& bs, uint32_t match_s, uint32_t r)
{
    const uint32_t m = lds32c(match_s + r * 4u);
    bs.put(m & 0xFFFFFFu, m >> 24);
}
template <int POS>
__device__ __forceinline__ uint32_t flit_off(uint32_t w, uint32_t nb)
{
    const uint32_t x = POS == 0 ? (w << 2) : (POS == 1 ? (w >> 6) : (POS == 2 ? (w >> 14) : (w >> 22)));
    return (x & 0x3FCu) | nb;
}
__device__ __forceinline__ void fput_word(LaneStager& bs, uint32_t lit_s, uint32_t w, uint32_t nb)
{
    const uint32_t nb8 = nb << 1;                                            // null half of the 8-byte table
    const uint32_t l64 = lit_s - 4096u;                                       // the 8-byte table sits directly below the 4-byte one
    const uint2 e0 = lds64c(l64 + flit_off8<0>(w, nb8)), e1 = lds64c(l64 + flit_off8<1>(w, nb8));
    const uint2 e2 = lds64c(l64 + flit_off8<2>(w, nb8)), e3 = lds64c(l64 + flit_off8<3>(w, nb8));
    fput_pair2(bs, e0, e1);
    fput_pair2(bs, e2, e3);
}
// the 4 literal codes of a word whose bytes belong to two pixels: bytes [0, SPLIT) carry null flag nbA, bytes [SPLIT, 4) nbB
// (0 or 0x400: the all-zero half of the table switches a pixel's literals off without a branch)
template <int SPLIT>
__device__ __forceinline__ void fput_word_2nb(LaneStager& bs, uint32_t lit_s, uint32_t w, uint32_t nbA, uint32_t nbB)
{
    const uint32_t l64 = lit_s - 4096u, a8 = nbA << 1, b8 = nbB << 1;
    const uint2 e0 = lds64c(l64 + flit_off8<0>(w, SPLIT > 0 ? a8 : b8)), e1 = lds64c(l64 + flit_off8<1>(w, SPLIT > 1 ? a8 : b8));
    const uint2 e2 = lds64c(l64 + flit_off8<2>(w, SPLIT > 2 ? a8 : b8)), e3 = lds64c(l64 + flit_off8<3>(w, SPLIT > 3 ? a8 : b8));
    fput_pair2(bs, e0, e1);
    fput_pair2(bs, e2, e3);
}

template <int CHANS>
__device__ __forceinline__ void fput_literal(LaneStager& bs, uint32_t lit_s, uint32_t px)
{
    fput_pair(bs, lds32c(lit_s + flit_off<0>(px, 0u)), lds32c(lit_s + flit_off<1>(px, 0u)));
    if (CHANS == 4) fput_pair(bs, lds32c(lit_s + flit_off<2>(px, 0u)), lds32c(lit_s + flit_off<3>(px, 0u)));
    else { const uint32_t c2 = lds32c(lit_s + flit_off<2>(px, 0u)); bs.put(c2 & 0xFFFFu, c2 >> 16); }
}
template <uint32_t M>
__device__ __forceinline__ uint32_t frun_before(uint32_t eqm, uint32_t r_in, uint32_t kk)
{
    const uint32_t t = ~eqm & ((1u << kk) - 1u);
    if (t == 0u) { const uint32_t r = kk + r_in; return r >= M ? r - M : r; }
    return kk - 1u - (31u - (uint32_t)__clz((int)t));
}

struct GroupDesc {                                // 32 bytes per row group; zeroed before every launch
    unsigned long long agg;                       // [63:62] 0 empty / 1 aggregate / 2 inclusive, [61:0] bits (aggregate) or end bit position (inclusive)
    unsigned long long tail;                      // bit 63 ready; low 32 bits: the partial word this group shares with its successor
    unsigned long long crc;                       // low 32 bits: raw CRC of the group's bit string zero-padded to whole words; high 32: those words
    unsigned long long pad_;
};

struct FusedParams {
    const uint8_t* pixels; size_t image_stride; uint32_t w, h;
    const CodeBook* books; uint32_t book_stride;
    uint2* row_adler; ImageState* st;
    GroupDesc* desc; uint32_t* ticket;
    uint32_t rows_per_group, steps_per_row, groups_per_image, n_images;
    uint8_t* out; size_t out_stride;
    uint32_t merge_first_unit;
};

template <int CHANS, bool DIRECT>
__global__ void __launch_bounds__(32 * kFusedWarps, CHANS == 3 ? 4 : 3) encode_fused_kernel(FusedParams p)
{
    using WK = typename FusedLoader<CHANS, DIRECT>::type;
    constexpr uint32_t M = max_match_pixels(CHANS);
    constexpr int kHalfWords = 2 * CHANS;
    constexpr int kUnitBytes = fused_unit_bytes<CHANS, DIRECT>();
    constexpr int kSlotWords = fused_slot_words<CHANS>();
    constexpr int kUnitWords = fused_unit_words<CHANS>();
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    // layout: [units: tile / lane-local strings][staging words][lit 512][match 88][small]
    const uint32_t nwarps = blockDim.x >> 5;
    uint32_t* s_stage = reinterpret_cast<uint32_t*>(dyn_smem + kFusedWarps * kUnitBytes);
    const uint32_t stage_words = kFusedWarps * kUnitWords + 2;
    uint32_t* s_lit64 = s_stage + stage_words;      // [512][2]: (code, size) pairs + the all-zero null half, directly below s_lit
    uint32_t* s_lit = s_lit64 + 1024;
    uint32_t* s_match = s_lit + 512;
    uint32_t* s_small = s_match + 88;               // 48 words
    // s_small: [0..7] has_lit, [8..15] trail, [16..23] npix, [24..31] unit bits, [32] ticket, [33] pred tail, [34] sh, [35] status
    unsigned long long* s_u64 = reinterpret_cast<unsigned long long*>(s_small + 48);     // [0..7] adler A, [8..15] adler B, [16] base (file bit of the group's first bit)

    const uint32_t lane = threadIdx.x & 31, warp = __shfl_sync(kFullMask, threadIdx.x >> 5, 0), tid = threadIdx.x;
    // Row groups are processed in stream order.  CTAs of a 1-D grid are dispatched in blockIdx order on every NVIDIA GPU (the
    // decoupled look-back of CUB's device-wide scan relies on the same property), so a group only waits for groups that are
    // already resident; FPNGB_FUSED_TICKET=1 (build flag) switches to an atomic ticket, which does not depend on that.
#if FPNGB_FUSED_TICKET
    if (tid == 0) s_small[32] = atomicAdd(p.ticket, 1u);
    for (uint32_t i = tid; i < stage_words; i += blockDim.x) s_stage[i] = 0u;
    __syncthreads();
    const uint32_t ticket = s_small[32];
#else
    for (uint32_t i = tid; i < stage_words; i += blockDim.x) s_stage[i] = 0u;
    const uint32_t ticket = blockIdx.x;
#endif
    const uint32_t img = ticket / p.groups_per_image, g = ticket - img * p.groups_per_image;
    if (img >= p.n_images) return;
    const CodeBook* book = p.books + (size_t)img * p.book_stride;
    for (uint32_t i = tid; i < 256; i += blockDim.x) {
        const uint32_t e = book->lit[i];
        s_lit[i] = e; s_lit[256 + i] = 0u;
        s_lit64[2 * i] = e & 0xFFFFu; s_lit64[2 * i + 1] = e >> 16; s_lit64[512 + 2 * i] = 0u; s_lit64[512 + 2 * i + 1] = 0u;
    }
    if (tid < 88) s_match[tid] = book->match[tid];
    uint32_t* s_crc = reinterpret_cast<uint32_t*>(s_u64 + 18);                // [4][256] slice tables of the 128-byte advance
    for (uint32_t i = tid; i < 1024; i += blockDim.x) s_crc[i] = (&g_f128b[0][0])[i];

    const uint32_t w = p.w, bpl = w * CHANS, S = p.steps_per_row;
    const uint32_t r_in_group = warp / S, step = warp - r_in_group * S;
    const uint32_t y = g * p.rows_per_group + r_in_group;
    const bool active = r_in_group < p.rows_per_group && y < p.h;
    uint8_t* unit_mem = dyn_smem + warp * kUnitBytes;
    const uint32_t lit_s = smem_u32(s_lit), match_s = smem_u32(s_match);

    // ---- phase 1: load, filter, Adler, equality
    uint32_t dw[WK::kWords];
    uint32_t eqm = 0, litm = 0, nvp = 0, trail = 0, has_lit_ballot = 0;
    bool last = false;
    uint32_t sumA = 0; unsigned long long sumB = 0;
    const uint8_t* cur = nullptr; const uint8_t* prev = nullptr;
    const uint32_t p0 = step * kStep16 + lane * kPix16;
    if (active) {
        cur = p.pixels + (size_t)img * p.image_stride + (size_t)y * bpl;
        prev = y ? cur - bpl : nullptr;
        WK wk; wk.init(lane, unit_mem);
        wk.bind(cur, prev);
        wk.prefetch(cur, prev, step, bpl, lane, unit_mem);
        // the filtered pixel left of this unit (lane 0 only needs it): a few byte loads that overlap the tile copy
        uint32_t left_px = 0;
        if (lane == 0 && step > 0) {
            const uint32_t o = (p0 - 1u) * CHANS;
#pragma unroll
            for (int b = 0; b < CHANS; b++) {
                const uint32_t cv = ld_u8(cur + o + b), pv = prev ? ld_u8(prev + o + b) : 0u;
                left_px |= ((cv - pv) & 0xFFu) << (8 * b);
            }
        }
        wk.template consume<true>(prev != nullptr, 0u, step, bpl, lane, unit_mem, dw, sumA, sumB);
        uint32_t px[16];
        WK::pixels(dw, px);
        nvp = p0 < w ? min(16u, w - p0) : 0u;
        uint32_t left = __shfl_up_sync(kFullMask, px[15], 1);
        if (lane == 0) left = left_px;
        uint32_t eq = (p0 > 0 && px[0] == left) ? 1u : 0u;
#pragma unroll
        for (int k = 1; k < 16; k++) eq |= (px[k] == px[k - 1]) ? (1u << k) : 0u;
        const uint32_t valid = (1u << nvp) - 1u;
        eqm = eq & valid;
        litm = valid & ~eq;
        last = nvp > 0 && p0 + nvp == w;
        trail = litm ? (nvp - 1u - (31u - (uint32_t)__clz((int)litm))) : nvp;
        has_lit_ballot = __ballot_sync(kFullMask, litm != 0);
        // what the units to the right need to know about this one
        const uint32_t npix = min(kStep16, w - step * kStep16);
        if (has_lit_ballot) {
            const uint32_t hl = 31u - (uint32_t)__clz((int)has_lit_ballot);
            const uint32_t t_hl = __shfl_sync(kFullMask, trail, hl), n_hl = __shfl_sync(kFullMask, nvp, hl);
            if (lane == 0) { s_small[warp] = 1u; s_small[8 + warp] = t_hl + npix - 16u * hl - n_hl; s_small[16 + warp] = npix; }
        } else if (lane == 0) { s_small[warp] = 0u; s_small[8 + warp] = npix; s_small[16 + warp] = npix; }
        // Adler partials of the unit
        const unsigned long long A = warp_sum_u64(sumA), B = warp_sum_u64(sumB);
        if (lane == 0) { s_u64[warp] = A; s_u64[8 + warp] = B; }
    }
    __syncthreads();                                                         // #1: tables, unit run info

    // ---- phase 2: tokenise + emit into the lane-local bit string
    uint32_t lane_bits = 0;
    const uint32_t slot_s = smem_u32(unit_mem) + lane * (kSlotWords * 4);
    if (active) {
        // run phase entering the unit: equal pixels that directly precede it, counted from the run's start (mod M)
        uint32_t run_in = 0;
        for (int t = (int)step - 1; t >= 0; t--) {
            const uint32_t u = r_in_group * S + (uint32_t)t;
            if (s_small[u]) { run_in += s_small[8 + u]; break; }
            run_in += s_small[16 + u];
        }
        run_in %= M;
        const uint32_t lower = has_lit_ballot & ((1u << lane) - 1u);
        const uint32_t src = lower ? (31u - (uint32_t)__clz((int)lower)) : 0u;
        const uint32_t src_trail = __shfl_sync(kFullMask, trail, src);
        const uint32_t r_lane = (lower ? (src_trail + 16u * (lane - src - 1u)) : (run_in + 16u * lane)) % M;

        const uint32_t lead = (uint32_t)__ffs((int)~eqm) - 1u;
        const uint32_t kM = M - 1u - r_lane;
        const uint32_t evm = (litm & ((eqm << 1) | (r_lane ? 1u : 0u))) | (kM < lead ? (1u << kM) : 0u);

        LaneStager bs; bs.begin(slot_s);
        if (lane == 0 && step == 0) { const uint32_t fcode = s_lit[y ? 2 : 0]; bs.put(fcode & 0xFFFFu, fcode >> 16); }
#pragma unroll 1
        for (uint32_t hh = 0; hh < 2; hh++) {
            const uint32_t lit8 = (litm >> (8u * hh)) & 0xFFu, ev8 = (evm >> (8u * hh)) & 0xFFu;
            uint32_t hw[kHalfWords];
#pragma unroll
            for (int j = 0; j < kHalfWords; j++) hw[j] = hh ? dw[kHalfWords + j] : dw[j];
            if (__all_sync(kFullMask, lit8 == 0xFFu && ev8 == 0u)) {
#pragma unroll
                for (int j = 0; j < kHalfWords; j++) fput_word(bs, lit_s, hw[j], 0u);
            } else if (__all_sync(kFullMask, lit8 == 0u)) {
                if (ev8) fput_match(bs, match_s, M);
            } else if (__reduce_add_sync(kFullMask, (uint32_t)__popc(lit8)) >= 16u) {
                const uint32_t nl = ~lit8;
                if (CHANS == 4) {
#pragma unroll
                    for (int k = 0; k < 8; k++) {
                        if (ev8 & (1u << k)) {
                            const uint32_t kk = 8u * hh + k;
                            const uint32_t len = ((eqm >> kk) & 1u) ? M : frun_before<M>(eqm, r_lane, kk);
                            if (len) fput_match(bs, match_s, len);
                        }
                        const uint32_t nb = (k <= 10 ? (nl << (10 - k)) : (nl >> (k - 10))) & 0x400u;
                        fput_word(bs, lit_s, hw[k % kHalfWords], nb);
                    }
                } else {
                    // RGB: the half's 24 filtered bytes as 6 words; word j holds bytes of pixels (4j)/3 .. (4j+3)/3.  A pixel's
                    // literals are switched off through the table's null half; the rare run tokens (at most a few per warp
                    // step) are inserted by a byte-wise emission of the one word in which the token's pixel starts.
#pragma unroll
                    for (int j = 0; j < 6; j++) {
                        constexpr int kFirstPx[6] = {0, 1, 2, 4, 5, 6};     // pixel of the word's first byte
                        constexpr int kSplit[6] = {3, 2, 1, 3, 2, 1};       // bytes of that pixel inside the word
                        constexpr uint32_t kStarts[6] = {0x03u, 0x04u, 0x08u, 0x30u, 0x40u, 0x80u};   // pixels whose first byte lies in the word
                        const int pa = kFirstPx[j];
                        const uint32_t wj = hw[j % kHalfWords];
                        if (ev8 & kStarts[j]) {
#pragma unroll
                            for (int i = 0; i < 4; i++) {
                                const int bidx = 4 * j + i, px = bidx / 3;
                                if (bidx % 3 == 0 && (ev8 & (1u << px))) {
                                    const uint32_t kk = 8u * hh + px;
                                    const uint32_t len = ((eqm >> kk) & 1u) ? M : frun_before<M>(eqm, r_lane, kk);
                                    if (len) fput_match(bs, match_s, len);
                                }
                                if (lit8 & (1u << px)) { const uint32_t e = lds32c(lit_s + (((wj >> (8 * i)) & 0xFFu) << 2)); bs.put(e & 0xFFFFu, e >> 16); }
                            }
                        } else {
                            const uint32_t nbA = (nl << (10 - pa)) & 0x400u, nbB = (nl << (10 - (pa + 1))) & 0x400u;
                            if (kSplit[j] == 3) fput_word_2nb<3>(bs, lit_s, wj, nbA, nbB);
                            else if (kSplit[j] == 2) fput_word_2nb<2>(bs, lit_s, wj, nbA, nbB);
                            else fput_word_2nb<1>(bs, lit_s, wj, nbA, nbB);
                        }
                    }
                }
            } else {
                uint32_t r = frun_before<M>(eqm, r_lane, 8u * hh);
#pragma unroll 1
                for (uint32_t gq = 0; gq < 2; gq++) {
                    uint32_t q[4];
                    if (CHANS == 4) {
#pragma unroll
                        for (int j = 0; j < 4; j++) q[j] = gq ? hw[(4 + j) % kHalfWords] : hw[j];
                    } else {
                        const uint32_t w0 = gq ? hw[3] : hw[0], w1 = gq ? hw[4] : hw[1], w2 = gq ? hw[5 % kHalfWords] : hw[2];
                        q[0] = w0 & 0x00FFFFFFu;
                        q[1] = __byte_perm(w0, w1, 0x4543) & 0x00FFFFFFu;
                        q[2] = __byte_perm(w1, w2, 0x4432) & 0x00FFFFFFu;
                        q[3] = w2 >> 8;
                    }
                    const uint32_t e4 = eqm >> (8u * hh + 4u * gq), base4 = 8u * hh + 4u * gq;
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        if (base4 + j < nvp) {
                            if (e4 & (1u << j)) {
                                if (++r == M) { fput_match(bs, match_s, M); r = 0; }
                            } else {
                                if (r) { fput_match(bs, match_s, r); r = 0; }
                                fput_literal<CHANS>(bs, lit_s, q[j]);
                            }
                        }
                    }
                }
            }
        }
        if (last) {
            const uint32_t r = frun_before<M>(eqm, r_lane, nvp);
            if (r) fput_match(bs, match_s, r);
            if (y == p.h - 1) {
                // capacity rule (SURVEY Q5): bits of the image's last flush unit; then the end-of-block code (fpng.cpp:1249)
                const uint32_t k = nvp - 1u;
                uint32_t lu;
                if (litm & (1u << k)) {
                    uint32_t px[16];
                    WK::pixels(dw, px);
                    uint32_t lastpx = px[0];
#pragma unroll
                    for (int q = 1; q < 16; q++) lastpx = (k == (uint32_t)q) ? px[q] : lastpx;
                    lu = (s_lit[lastpx & 0xFFu] >> 16) + (s_lit[(lastpx >> 8) & 0xFFu] >> 16) + (s_lit[(lastpx >> 16) & 0xFFu] >> 16);
                    if (CHANS == 4) lu += s_lit[lastpx >> 24] >> 16;
                    if (w == 1 && p.merge_first_unit) lu += s_lit[y ? 2 : 0] >> 16;
                } else lu = r ? (s_match[r] >> 24) : (s_match[M] >> 24);
                p.st[img].last_unit_bits = lu;
                bs.put(book->eob & 0xFFFFu, book->eob >> 16);
            }
        }
        lane_bits = bs.finish();
    }
    // ---- phase 3: bit offsets (lane in unit, unit in group, group in file)
    uint32_t unit_bits = 0;
    const uint32_t lane_ofs = warp_excl_scan_u32(lane_bits, lane, unit_bits);
    if (lane == 0) s_small[24 + warp] = unit_bits;
    __syncthreads();                                                         // #2: unit bit counts, lane strings complete
    uint32_t unit_ofs = 0, group_bits = 0;
    for (uint32_t u = 0; u < nwarps; u++) { const uint32_t b = s_small[24 + u]; if (u < warp) unit_ofs += b; group_bits += b; }

    GroupDesc* desc = p.desc + (size_t)img * p.groups_per_image;
    if (warp == 0) {
        // publish this group's bit count at once: later groups can already sum it while this one is still busy
        if (g != 0 && lane == 0) st_volatile_u64(&desc[g].agg, ((unsigned long long)kStateAgg << 62) | group_bits);
        // Adler-32 partials per scanline (rows of this group; their units are this CTA's warps)
        if (lane < p.rows_per_group && g * p.rows_per_group + lane < p.h) {
            unsigned long long A = 0, B = 0;
            for (uint32_t t = 0; t < S; t++) { A += s_u64[lane * S + t]; B += s_u64[8 + lane * S + t]; }
            const uint32_t yy = g * p.rows_per_group + lane, filt = yy ? 2u : 0u;
            const unsigned long long n = (unsigned long long)bpl + 1ull, S1 = A + filt, S2 = n * S1 - (A + B);
            p.row_adler[(size_t)img * p.h + yy] = make_uint2((uint32_t)(S1 % kAdlerMod), (uint32_t)(S2 % kAdlerMod));
        }
    }

    // ---- phase 4a: every lane copies its bit string into the CTA staging buffer (group-relative bit positions)
    if (active && lane_bits) {
        const uint32_t o = unit_ofs + lane_ofs, sh = o & 31u, nw = (lane_bits + 31u) >> 5;
        const uint32_t stage_s = smem_u32(s_stage) + ((o >> 5) << 2);
        uint32_t prevw = 0;
        for (uint32_t k = 0; k <= nw; k++) {
            const uint32_t v = k < nw ? lds32(slot_s + k * 4u) : 0u;
            const uint32_t outw = __funnelshift_l(prevw, v, sh);             // (v << sh) | (prevw >> (32 - sh)); sh == 0 -> v
            prevw = v;
            // the word is exclusively this lane's when the lane's string covers all 32 of its bits
            const bool whole = k >= 1u && (k << 5) + 32u <= sh + lane_bits;
            if (whole) sts32(stage_s + k * 4u, outw);
            else if (outw) red_or32(stage_s + k * 4u, outw);
        }
    }
    __syncthreads();                                                         // #3: staging complete
    const uint32_t NWc = (group_bits + 31u) >> 5;
    if (warp == 0) {
        // decoupled look-back (single-pass chained scan) while the other warps compute the CRC partial: sum the aggregates of
        // the groups before, stop at the first group that already knows its inclusive end position
        unsigned long long base = 0;
        uint32_t status = 0;
        if (g == 0) {
            base = (unsigned long long)kZlibBitBase + book->hdr_bits;
        } else {
            int j = (int)g - 1;
            bool done = false;
            uint32_t spins = 0;
            while (!done) {
                const int idx = j - (int)lane;
                unsigned long long v = idx >= 0 ? ld_volatile_u64(&desc[idx].agg) : ((unsigned long long)kStateIncl << 62);   // before group 0: nothing
                const uint32_t state = (uint32_t)(v >> 62);
                const uint32_t incl = __ballot_sync(kFullMask, state == kStateIncl);
                const uint32_t empty = __ballot_sync(kFullMask, state == 0u);
                const uint32_t first = incl ? (uint32_t)__ffs((int)incl) - 1u : 32u;       // nearest group with an inclusive value
                const uint32_t needed = first >= 31u ? kFullMask : ((2u << first) - 1u);   // lanes whose value enters the sum
                if (empty & needed) {                                       // a predecessor that matters has not published yet: look again
                    if (++spins > kSpinLimit) { status = 1u; break; }
                    __nanosleep(200);                                       // leave the issue slots to the CTAs that still have work
                    continue;
                }
                unsigned long long contrib = (lane <= first && idx >= 0) ? (v & kValueMask) : 0ull;
                contrib = warp_sum_u64(contrib);
                base += contrib;
                if (incl) done = true; else j -= 32;
            }
            // (lanes with idx < 0 report "inclusive 0" only to keep the ballot well defined: group 0 always publishes an
            //  inclusive value, so every chain ends at or before it)
        }
        const unsigned long long end = base + group_bits;
        if (lane == 0) {
            st_volatile_u64(&desc[g].agg, ((unsigned long long)kStateIncl << 62) | end);
            s_u64[16] = base;
            s_small[35] = status;
            // the word shared with the predecessor / successor.  This group's own trailing partial word (bits below span & 31
            // of word nfull) does not depend on the predecessor when the group completes at least one word (always, except
            // for degenerate tiny groups): it is published BEFORE waiting for the predecessor's, so the tails of consecutive
            // groups do not form a serial chain.
            const uint32_t sh = (uint32_t)(base & 31ull);
            const unsigned long long W0 = base >> 5;
            const uint32_t span = sh + group_bits, nfull = span >> 5;
            uint32_t tailw = 0;
            if (span & 31u) tailw = __funnelshift_l(nfull ? s_stage[nfull - 1] : 0u, s_stage[nfull], sh);
            if (nfull) st_volatile_u64(&desc[g].tail, kTailReady | tailw);
            uint32_t pred = 0;
            if (sh && !status) {
                if (g == 0) {
                    const uint32_t byte0 = (uint32_t)(W0 << 2) - kPngHeaderSize;  // always inside the block header bytes (hdr_bits > 64)
                    const uint32_t word = (uint32_t)book->hdr[byte0] | ((uint32_t)book->hdr[byte0 + 1] << 8) | ((uint32_t)book->hdr[byte0 + 2] << 16) | ((uint32_t)book->hdr[byte0 + 3] << 24);
                    pred = word & ((1u << sh) - 1u);
                } else {
                    unsigned long long t;
                    uint32_t spins = 0;
                    while (!((t = ld_volatile_u64(&desc[g - 1].tail)) & kTailReady) && ++spins < kSpinLimit) __nanosleep(100);
                    if (!(t & kTailReady)) p.st[img].status = 3u;
                    pred = (uint32_t)t;
                }
            }
            s_small[33] = pred;
            if (!nfull) st_volatile_u64(&desc[g].tail, kTailReady | tailw | pred);
        }
        if (lane == 0 && nwarps > 1) s_small[36] = 0u;
    }
    // ---- CRC-32 partial of the group's bit string (staging words, group-relative: independent of the file position); warp 0
    // is busy with the look-back unless it is the only warp
    if (warp != 0 || nwarps == 1) {
        const uint32_t cw = nwarps > 1 ? nwarps - 1u : 1u, first = nwarps > 1 ? warp - 1u : 0u;
        uint32_t acc = 0;
        // this warp takes the chunks first, first + cw, ... counted from the END of the string
        for (uint32_t m = first; m * kCrcChunkWords < NWc; m += cw) {
            const int j0 = (int)NWc - (int)((m + 1u) * kCrcChunkWords) + (int)lane;     // this lane's first word of the chunk (may be < 0: front padding)
            uint32_t c = 0;
#pragma unroll
            for (uint32_t k = 0; k < kCrcChunkWords / 32u; k++) {
                const int j = j0 + (int)(32u * k);
                const uint32_t x = c ^ (j >= 0 ? s_stage[j] : 0u);
                if (k + 1u < kCrcChunkWords / 32u)
                    c = s_crc[x & 0xFFu] ^ s_crc[256 + ((x >> 8) & 0xFFu)] ^ s_crc[512 + ((x >> 16) & 0xFFu)] ^ s_crc[768 + (x >> 24)];
                else c = x;
            }
            c = mul_nibbles(g_lane_mul[lane], c);                              // lane l's last word sits 31 - l words before the chunk end
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) c ^= __shfl_xor_sync(kFullMask, c, o);
            // position the chunk: m chunks follow it (lanes 0..7 look up one nibble each)
            uint32_t part = lane < 8u ? __ldg(&g_chunk_mul[m & 31u][lane][(c >> (4u * lane)) & 15u]) : 0u;
            part ^= __shfl_xor_sync(kFullMask, part, 4); part ^= __shfl_xor_sync(kFullMask, part, 2); part ^= __shfl_xor_sync(kFullMask, part, 1);
            acc ^= part;
        }
        if (lane == 0) s_small[36 + warp] = acc;
    }
    __syncthreads();                                                         // #4: base, pred tail, CRC partials
    const unsigned long long base = s_u64[16];
    const uint32_t sh = (uint32_t)(base & 31ull);
    const unsigned long long W0 = base >> 5;
    const uint32_t span = sh + group_bits, nfull = span >> 5;                // words whose bit 31 this group covers
    (void)span;
    if (s_small[35]) { if (tid == 0) p.st[img].status = 2u; return; }
    if (tid == 0) {
        uint32_t r = 0;
        for (uint32_t u = 0; u < nwarps; u++) r ^= s_small[36 + u];
        desc[g].crc = (unsigned long long)r | ((unsigned long long)NWc << 32);
    }
    // ---- phase 4c: write the complete words, shifted to the group's position in the file
    {
        uint32_t* gw = reinterpret_cast<uint32_t*>(p.out + (size_t)img * p.out_stride);
        const unsigned long long raw = ((unsigned long long)bpl + 1ull) * p.h;
        const unsigned long long cap_words = (((kPngHeaderSize + raw + 7ull) & ~7ull)) >> 2;   // the reference's buffer (fpng.cpp:1705): never write past it
        const uint32_t pred = s_small[33];
        for (uint32_t m = tid; m < nfull; m += blockDim.x) {
            uint32_t v = __funnelshift_l(m ? s_stage[m - 1] : 0u, s_stage[m], sh);
            if (m == 0) v |= pred;
            if (W0 + m < cap_words) gw[W0 + m] = v;
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Finishing kernel, one CTA per image: compressed-vs-stored decision with the reference's exact rule, container header,
// block header, the last partial word, IEND, stored-block headers, ImageState for the Adler / CRC kernels.
// ------------------------------------------------------------------------------------------------------------------
struct FinishParams {
    const GroupDesc* desc; uint32_t groups_per_image;
    const CodeBook* books; uint32_t book_stride;
    ImageState* st;
    uint8_t* out; size_t out_stride; uint32_t* sizes;
    uint32_t w, h, chans, flags;
    uint8_t png_header[kPngHeaderSize];
};

__global__ void __launch_bounds__(256) fused_finish_kernel(FinishParams p)
{
    const uint32_t img = blockIdx.x, tid = threadIdx.x;
    const CodeBook* book = p.books + (size_t)img * p.book_stride;
    ImageState* st = p.st + img;
    uint8_t* file = p.out + (size_t)img * p.out_stride;
    const GroupDesc last = p.desc[(size_t)img * p.groups_per_image + p.groups_per_image - 1];
    const uint32_t hdr_bits = book->hdr_bits, eob_size = book->eob >> 16;
    const unsigned long long end = last.agg & kValueMask;                   // file bit right after the end-of-block code
    const unsigned long long total_bits = end - kZlibBitBase;               // zlib bits incl. header and EOB
    const unsigned long long raw = ((unsigned long long)p.w * p.chans + 1ull) * p.h;
    const unsigned long long cap = ((kPngHeaderSize + raw + 7ull) & ~7ull) - kPngHeaderSize;      // fpng.cpp:1705
    const unsigned long long d_last = (total_bits - eob_size - st->last_unit_bits) >> 3;
    const unsigned long long zbytes = (total_bits + 7ull) >> 3;
    const bool sane = (last.agg >> 62) == kStateIncl && st->status == 0u;
    const bool compressed = sane && !(p.flags & 2u) && (d_last + 8ull <= cap) && (zbytes + 4ull <= cap);
    const unsigned long long nblk = (raw + 65534ull) / 65535ull;
    const uint32_t zsize = compressed ? (uint32_t)(zbytes + 4ull) : (uint32_t)(2ull + raw + 5ull * nblk + 4ull);

    const unsigned long long base = (unsigned long long)kZlibBitBase + hdr_bits;
    // header bytes: everything before the word that holds the first token bit (that word is written by row group 0)
    const uint32_t hbytes = compressed ? (hdr_bits + 7u) >> 3 : 2u;
    const uint32_t hend = compressed ? 4u * (uint32_t)(base >> 5) : kPngHeaderSize + 2u;
    for (uint32_t i = tid; i < hend; i += blockDim.x) {
        uint8_t v = 0;
        if (i < kPngHeaderSize) v = p.png_header[i];
        else if (i - kPngHeaderSize < hbytes) v = compressed ? book->hdr[i - kPngHeaderSize] : (i == kPngHeaderSize ? 0x78 : 0x01);
        if (i >= 50 && i < 54) v = (uint8_t)(zsize >> (8 * (53 - i)));
        file[i] = v;
    }
    if (!compressed) {
        for (unsigned long long j = tid; j < nblk; j += blockDim.x) {       // stored block headers (fpng.cpp:829-850)
            uint8_t* b = file + kPngHeaderSize + 2ull + j * 65540ull;
            const unsigned long long remaining = raw - j * 65535ull;
            const uint32_t len = remaining < 65535ull ? (uint32_t)remaining : 65535u;
            b[0] = (j + 1 == nblk) ? 1 : 0;
            b[1] = (uint8_t)len; b[2] = (uint8_t)(len >> 8);
            b[3] = (uint8_t)~len; b[4] = (uint8_t)(~len >> 8);
        }
    }
    if (tid == 0) {
        if (compressed && (end & 31ull)) {
            // the last, partial word of the token stream (EOB included); pad bits are zero (fpng.cpp:1249-1251)
            const uint32_t tw = (uint32_t)last.tail;
            uint8_t* q = file + ((end >> 5) << 2);
            const uint32_t nb = (uint32_t)(((end & 31ull) + 7ull) >> 3);
            for (uint32_t i = 0; i < nb; i++) q[i] = (uint8_t)(tw >> (8 * i));
        }
        static const uint8_t iend[12] = { 0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82 };
        uint8_t* t = file + kPngHeaderSize + zsize;
        for (int i = 0; i < 4; i++) t[i] = 0;
        for (int i = 0; i < 12; i++) t[4 + i] = iend[i];
        st->zsize = zsize;
        st->stored = compressed ? 0u : 1u;
        st->crc_acc = 0u;
        st->tiles_done = 0u;
        p.sizes[img] = kPngHeaderSize + zsize + kPngTrailerSize;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// CRC-32 of "IDAT" + zlib stream (fpng.cpp:1797-1800) from the per-group partials, one CTA per image.  With E = end of the
// message (file bit (58 + zsize) * 8), a piece that starts at file bit s and whose raw CRC covers nw words contributes
// raw * x^(E - s - 32 nw).  Pieces: the bytes/bits before the first token ("IDAT", zlib header, block header), the row
// groups, the four Adler-32 bytes.  Initial value and final XOR (0xFFFFFFFF) are applied by linearity.
// ------------------------------------------------------------------------------------------------------------------
struct FusedCrcParams {
    const GroupDesc* desc; uint32_t groups_per_image;
    const CodeBook* books; uint32_t book_stride;
    const ImageState* st;
    uint8_t* out; size_t out_stride;
};

__global__ void __launch_bounds__(256) fused_crc_kernel(FusedCrcParams p)
{
    __shared__ uint32_t s_part[8];
    const uint32_t img = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const ImageState st = p.st[img];
    if (st.stored || st.status) return;                                      // stored-block images: idat_crc_stream_kernel reads the file
    const CodeBook* book = p.books + (size_t)img * p.book_stride;
    const GroupDesc* desc = p.desc + (size_t)img * p.groups_per_image;
    const unsigned long long E = (unsigned long long)(kPngHeaderSize + st.zsize) * 8ull;
    const unsigned long long msg0 = (unsigned long long)(kPngHeaderSize - 4u) * 8ull, base0 = (unsigned long long)kZlibBitBase + book->hdr_bits;
    uint32_t acc = 0;
    for (uint32_t g = tid; g < p.groups_per_image; g += blockDim.x) {
        const unsigned long long c = desc[g].crc;
        const unsigned long long start = g ? (desc[g - 1].agg & kValueMask) : base0;
        const unsigned long long e = E - start - 32ull * (c >> 32);
        acc ^= gf2_mulmod((uint32_t)c, gf2_pow(c_fx_pow2, e));
    }
    if (tid == 0) {
        // "IDAT" + header bits, bit by bit (a few hundred to ~2400 bits), then shifted to the end of the message
        uint32_t reg = 0;
        const uint8_t tag[4] = {'I', 'D', 'A', 'T'};
        for (int i = 0; i < 32; i++) reg = crc_bit_step(reg, (tag[i >> 3] >> (i & 7)) & 1u);
        const uint32_t hb = book->hdr_bits;
        for (uint32_t i = 0; i < hb; i++) reg = crc_bit_step(reg, (book->hdr[i >> 3] >> (i & 7)) & 1u);
        acc ^= gf2_mulmod(reg, gf2_pow(c_fx_pow2, E - base0));
        // Adler-32, big-endian, last four bytes of the message
        uint32_t ra = 0;
        for (int i = 0; i < 32; i++) { const uint32_t byte = (st.adler >> (24 - 8 * (i >> 3))) & 0xFFu; ra = crc_bit_step(ra, (byte >> (i & 7)) & 1u); }
        acc ^= ra;
        // initial register value 0xFFFFFFFF advanced over the whole message, and the final XOR
        acc ^= gf2_mulmod(0xFFFFFFFFu, gf2_pow(c_fx_pow2, E - msg0)) ^ 0xFFFFFFFFu;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc ^= __shfl_xor_sync(0xFFFFFFFFu, acc, o);
    if (lane == 0) s_part[warp] = acc;
    __syncthreads();
    if (tid == 0) {
        uint32_t crc = 0;
        for (int i = 0; i < 8; i++) crc ^= s_part[i];
        uint8_t* q = p.out + (size_t)img * p.out_stride + kPngHeaderSize + st.zsize;
        q[0] = (uint8_t)(crc >> 24); q[1] = (uint8_t)(crc >> 16); q[2] = (uint8_t)(crc >> 8); q[3] = (uint8_t)crc;
    }
}

void launch_fused_crc(const void* desc_mem, uint32_t n, uint32_t w, uint32_t h, const CodeBook* books, uint32_t book_stride, const ImageState* st,
                      uint8_t* out, size_t out_stride, cudaStream_t s)
{
    const uint32_t S = (w + kStep16 - 1) / kStep16, R = kFusedWarps / S, G = (h + R - 1) / R;
    FusedCrcParams c{(const GroupDesc*)desc_mem, G, books, book_stride, st, out, out_stride};
    fused_crc_kernel<<<n, 256, 0, s>>>(c);
}

// ------------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------------
template <int CHANS, bool DIRECT> constexpr size_t fused_smem()
{
    return (size_t)kFusedWarps * fused_unit_bytes<CHANS, DIRECT>() + ((size_t)kFusedWarps * fused_unit_words<CHANS>() + 2 + 512 + 88 + 48 + 1024) * 4 + 18 * 8 + 1024 * 4 + 16;
}

bool fused_eligible(const void* base, size_t image_stride, uint32_t w, uint32_t h, uint32_t chans, uint32_t n)
{
    (void)base; (void)image_stride; (void)chans;             // any alignment: unaligned scanlines use the direct loader
    const uint32_t S = (w + kStep16 - 1) / kStep16;
    if (S > (uint32_t)kFusedWarps) return false;
    const uint32_t R = kFusedWarps / S;
    const unsigned long long groups = (unsigned long long)n * ((h + R - 1) / R);
    return groups < (1ull << 31);
}

size_t fused_desc_bytes(uint32_t n, uint32_t w, uint32_t h)
{
    const uint32_t S = (w + kStep16 - 1) / kStep16, R = kFusedWarps / S;
    return (size_t)n * ((h + R - 1) / R) * sizeof(GroupDesc) + 256;
}

// desc_mem: fused_desc_bytes() bytes (descriptors, then the ticket counter in the last 256 bytes)
int launch_encode_fused(const uint8_t* pixels, size_t image_stride, uint32_t n, uint32_t w, uint32_t h, uint32_t chans, uint32_t flags,
                        const CodeBook* books, uint32_t book_stride, uint2* row_adler, ImageState* st, void* desc_mem,
                        uint8_t* out, size_t out_stride, uint32_t* sizes, const uint8_t* png_header, uint32_t merge_first_unit, cudaStream_t s,
                        cudaEvent_t mid_event)
{
    const uint32_t S = (w + kStep16 - 1) / kStep16, R = kFusedWarps / S, G = (h + R - 1) / R;
    const size_t dbytes = (size_t)n * G * sizeof(GroupDesc);
    FPNGB_CUDA_OK(cudaMemsetAsync(desc_mem, 0, dbytes + 256, s));
    FPNGB_CUDA_OK(cudaMemsetAsync(st, 0, (size_t)n * sizeof(ImageState), s));
    FusedParams p{};
    p.pixels = pixels; p.image_stride = image_stride; p.w = w; p.h = h; p.books = books; p.book_stride = book_stride;
    p.row_adler = row_adler; p.st = st; p.desc = (GroupDesc*)desc_mem; p.ticket = (uint32_t*)((uint8_t*)desc_mem + dbytes);
    p.rows_per_group = R; p.steps_per_row = S; p.groups_per_image = G; p.n_images = n; p.out = out; p.out_stride = out_stride;
    p.merge_first_unit = merge_first_unit;
    const uint32_t threads = 32u * R * S;
    const unsigned long long groups = (unsigned long long)n * G;
    const bool direct = !walk16_eligible(pixels, image_stride, w * chans, w, chans);
#define FPNGB_LAUNCH_FUSED(C, D) do { FPNGB_SET_SMEM((encode_fused_kernel<C, D>), (fused_smem<C, D>())); \
        encode_fused_kernel<C, D><<<(uint32_t)groups, threads, fused_smem<C, D>(), s>>>(p); } while (0)
    if (chans == 4) { if (direct) FPNGB_LAUNCH_FUSED(4, true); else FPNGB_LAUNCH_FUSED(4, false); }
    else { if (direct) FPNGB_LAUNCH_FUSED(3, true); else FPNGB_LAUNCH_FUSED(3, false); }
#undef FPNGB_LAUNCH_FUSED
    if (mid_event) cudaEventRecord(mid_event, s);                            // profiling: end of the fused kernel
    FinishParams f{};
    f.desc = (const GroupDesc*)desc_mem; f.groups_per_image = G; f.books = books; f.book_stride = book_stride; f.st = st;
    f.out = out; f.out_stride = out_stride; f.sizes = sizes; f.w = w; f.h = h; f.chans = chans; f.flags = flags;
    memcpy(f.png_header, png_header, kPngHeaderSize);
    fused_finish_kernel<<<n, 256, 0, s>>>(f);
    return 0;
}

}  // namespace fpngb
