// fpng_b200/csrc/encode16_kernels.cu -- scan (K1) and pack (K3) kernels of the two-kernel encoder on the 16-pixels-per-lane
// walker (row_walk16.cuh), for every shape, alignment and layout.  K2 and the Adler-32 finalize are in encode_kernels.cu.
// LIT1: the RGBA 1-pass instantiations under a table whose "one-pixel match vs four literals" rule can fire (fpng.cpp:1520-1528).
#include "row_walk16.cuh"
#include "kernels.cuh"

namespace fpngb {

constexpr int kScan16Rows = 8;                   // warps (scanlines) per CTA, scan
// warps (scanline sequences) per CTA, pack: 8 for RGB, 7 for RGBA.  Shared memory per warp (tiles + staging) sets the CTAs per SM:
// RGB 4 x 7 or 3 x 8 warps, RGBA 3 x 7 or 2 x 8.  RGB runs faster with 8 (H100 at 700 W, C2: pack 1.54 against 1.64 ms, DESIGN 4.1).
__host__ __device__ constexpr int pack16_warps(int chans) { return chans == 4 ? 7 : 8; }
constexpr uint32_t kRowsPerWarp16 = 5;           // consecutive scanlines per warp (pack kernel) on large batches: amortises the CTA prologue and
                                                 // lets a scanline's first tile be prefetched during the previous scanline's last step
// small jobs (a single image) keep one scanline per warp so that the grid still fills the GPU
static uint32_t g_rows_per_warp_override = 0;    // tests force both shapes of the kernels on small inputs (fpngb_debug_rows_per_warp)
void set_rows_per_warp16(uint32_t v) { g_rows_per_warp_override = v > 64u ? 64u : v; }
static uint32_t sm_count()                       // the current device's SMs (132 on an H100 SXM), read once
{
    static uint32_t n = 0;
    if (!n) {
        int dev = 0, v = 0;
        if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && v > 0)
            n = (uint32_t)v;
        else
            n = 132u;
    }
    return n;
}
static uint32_t rows_per_warp16(uint32_t n, uint32_t h)
{
    if (g_rows_per_warp_override) return g_rows_per_warp_override;
    return (size_t)n * h >= (size_t)sm_count() * 64u * kRowsPerWarp16 ? kRowsPerWarp16 : 1u;
}
// staging words per warp step: lead-in (31) + filter literal (12) + 512 pixel slots of [pending match 18 bits][literal 12*CHANS bits]
template <int CHANS> __host__ __device__ constexpr int stage16_words() { return ((31 + 12 + 512 * (18 + 12 * CHANS)) / 32 + 1 + 15) / 16 * 16; }

__device__ __forceinline__ uint32_t byte1(uint32_t v) { return __byte_perm(v, 0u, 0x4441); }   // (v >> 8) & 0xFF in one PRMT
__device__ __forceinline__ uint32_t byte2(uint32_t v) { return __byte_perm(v, 0u, 0x4442); }

// scanline loader: staged tiles (TMA / cp.async) for 16-byte aligned interleaved scanlines, direct realigning 128-bit loads for
// any other interleaved shape, per-plane loads for planar images (ScanParams::chan_stride != 0); kLoad16* in kernels.cuh
template <int CHANS, int LOAD> struct Loader16 { using type = Walk16<CHANS>; };
template <int CHANS> struct Loader16<CHANS, kLoad16Direct> { using type = Walk16Direct<CHANS>; };
template <int CHANS> struct Loader16<CHANS, kLoad16Planar> { using type = Walk16Planar<CHANS>; };
template <class WK> __device__ __forceinline__ void set_planes(WK&, size_t) {}
template <int CHANS> __device__ __forceinline__ void set_planes(Walk16Planar<CHANS>& wk, size_t chan_stride) { wk.planes(chan_stride); }

template <int CHANS>
__device__ __forceinline__ uint32_t literal_bits16(const uint8_t* s_lit, uint32_t px)
{
    uint32_t b = s_lit[px & 0xFFu] + s_lit[byte1(px)];
    if (CHANS == 4) b += s_lit[byte2(px)] + s_lit[px >> 24];
    else b += s_lit[px >> 16];
    return b;
}

// RGBA pixel k - 1 of a lane (its words are its pixels), `left` (the pixel left of the lane) for k == 0
template <int N>
__device__ __forceinline__ uint32_t pixel_before16(const uint32_t (&px)[N], uint32_t left, uint32_t k)
{
    uint32_t v = left;
#pragma unroll
    for (int q = 0; q < N; q++) v = k == (uint32_t)q + 1u ? px[q] : v;
    return v;
}

// bits of a pending run of r pixels flushed before lane pixel k.  LIT1: a one-pixel match costs min(match, the four literals of
// the pixel it covers); the literals are taken iff the match costs more (fpng.cpp:1520-1528)
template <bool LIT1>
__device__ __forceinline__ uint32_t run_bits16(const uint8_t* s_lit, const uint8_t* s_match, uint32_t r, const uint32_t (&px)[16], uint32_t left,
                                               uint32_t k)
{
    const uint32_t b = s_match[r];
    if (!LIT1 || r != 1u) return b;
    return min(b, literal_bits16<4>(s_lit, pixel_before16(px, left, k)));
}

// Ragged launches (RAGGED = true): CTA blockIdx.x is CTA `cta` of one image (ragged_locate); the image's descriptor replaces the
// call-wide pixels, strides, shape and books, and the row / lane tables, image state and output are rebased to it, so that the
// kernel bodies run as for image 0 of a uniform batch.  The uniform instantiations compile without any of this.  Returns the
// image's index in the descriptor table.
template <class P>
__device__ __forceinline__ uint32_t ragged_image16(P& p, uint32_t& cta)
{
    const uint32_t i = ragged_locate(p.ragged, blockIdx.x, cta);
    const ImageDesc& d = p.ragged.desc[i];
    p.pixels = d.pixels; p.image_stride = 0; p.row_pitch = d.row_pitch; p.chan_stride = d.chan_stride; p.w = d.w; p.h = d.h;
    p.books = d.book; p.book_stride = 0;
    p.row_bits += d.row_base; p.row_adler += d.row_base; p.st += i;
    p.lane_ofs += d.lane_base; p.lane_ofs_pitch = d.lane_pitch;
    return i;
}

// ------------------------------------------------------------------------------------------------
// K1 (v2): per-row bit count + Adler partials (+ per-lane bit offsets inside the row for the pack kernel)
// ------------------------------------------------------------------------------------------------
// No minimum CTAs per SM: a bound of 5 (48 registers for RGB, 40 instead of 32 warps per SM) measured slower, since the kernel is
// ALU-pipe bound, not latency bound.
template <int CHANS, int LOAD, bool RAGGED = false, bool LIT1 = false>
__global__ void __launch_bounds__(32 * kScan16Rows) row_scan16_kernel(std::conditional_t<RAGGED, RaggedParams<ScanParams>, ScanParams> p)
{
    static_assert(!LIT1 || CHANS == 4, "the one-pixel-match rule is RGBA only");
    using WK = typename Loader16<CHANS, LOAD>::type;
    constexpr uint32_t M = max_match_pixels(CHANS);
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    uint8_t* s_lit = dyn_smem + kScan16Rows * WK::kWarpBytes;
    uint8_t* s_match = s_lit + 256;

    // the warp index as a shuffle result: the compiler then treats everything derived from it (scanline pointers, tile address) as
    // warp-uniform and issues the TMA copies from uniform registers without a per-lane "waterfall" loop
    const uint32_t lane = threadIdx.x & 31, warp = __shfl_sync(kFullMask, threadIdx.x >> 5, 0);
    uint32_t img = blockIdx.y, cta = blockIdx.x;
    if constexpr (RAGGED) { ragged_image16(p, cta); img = 0; }
    const uint32_t y = cta * kScan16Rows + warp;
    const CodeBook* book = p.books + (size_t)img * p.book_stride;
    static_assert(32 * kScan16Rows == 256, "one table byte per thread");
    s_lit[threadIdx.x] = book->lit_size[threadIdx.x];
    if (threadIdx.x < 88) s_match[threadIdx.x] = book->match_bits[threadIdx.x];
    __syncthreads();
    if (y >= p.h) return;

    const uint32_t w = p.w, bpl = w * CHANS;
    const uint8_t* cur = p.pixels + (size_t)img * p.image_stride + (size_t)y * p.row_pitch;
    const uint8_t* prev = y ? cur - p.row_pitch : nullptr;
    const uint32_t filt = y ? 2u : 0u;
    const uint32_t nsteps = (w + kStep16 - 1) / kStep16;
    uint8_t* tiles = dyn_smem + warp * WK::kWarpBytes;
    uint2* lane_ofs = p.lane_ofs + ((size_t)img * p.h + y) * p.lane_ofs_pitch;

    WK wk; wk.init(lane, tiles); wk.bind(cur, prev); set_planes(wk, p.chan_stride);
    RowCarry carry = {0u, 0u};
    uint32_t row_run = s_lit[filt];              // bits of the row emitted before the current step (filter literal first)
    uint32_t sumA = 0, last_unit = 0;
    unsigned long long sumB = 0;

    wk.prefetch(cur, prev, 0, bpl, lane, tiles);
    for (uint32_t step = 0; step < nsteps; step++) {
        uint32_t dw[WK::kWords], px[16];
        wk.template consume<true>(prev != nullptr, step, step, bpl, lane, tiles, dw, sumA, sumB);
        if (step + 1 < nsteps) wk.prefetch(cur, prev, step + 1, bpl, lane, tiles);         // lands while this step is processed
        WK::pixels(dw, px);
        const uint32_t p0 = step * kStep16 + lane * kPix16;
        uint32_t left = 0;                       // LIT1: the pixel left of the lane's first, which a run entering the lane covers
        if constexpr (LIT1) {
            left = __shfl_up_sync(kFullMask, px[15], 1);
            if (lane == 0) left = carry.prev_px;
        }
        const Lane16 t = classify16<CHANS>(px, p0, w, carry, lane);

        uint32_t bits = 0;
        // literal pixels: sum of code sizes.  Warp-uniform fast paths: no literal at all (RLE rows) / all literal (noisy rows)
        const uint32_t any_lit = __any_sync(kFullMask, t.litm != 0);
        if (any_lit) {
            if (__all_sync(kFullMask, t.litm == 0xFFFFu)) {
#pragma unroll
                for (int k = 0; k < 16; k++) bits += literal_bits16<CHANS>(s_lit, px[k]);
            } else {
                // mixed step: the per-pixel sizes (<= 48) of four pixels packed into one word (IMADs) and added under the literal mask
                // by ONE dp4a against the nibble spread to 0/1 bytes -- instead of three ALU-pipe mask instructions per pixel
                const uint32_t k8 = c_fma_k[2], k16 = c_fma_k[3], k24 = c_fma_k[4];
#pragma unroll
                for (int g = 0; g < 4; g++) {
                    const uint32_t c0 = literal_bits16<CHANS>(s_lit, px[4 * g]), c1 = literal_bits16<CHANS>(s_lit, px[4 * g + 1]);
                    const uint32_t c2 = literal_bits16<CHANS>(s_lit, px[4 * g + 2]), c3 = literal_bits16<CHANS>(s_lit, px[4 * g + 3]);
                    const uint32_t packed = c3 * k24 + (c2 * k16 + (c1 * k8 + c0));
                    const uint32_t m01 = (((t.litm >> (4 * g)) & 0xFu) * 0x00204081u) & 0x01010101u;   // bit j of the nibble -> byte j
                    bits = __dp4a(packed, m01, bits);
                }
            }
        }
        // match tokens: walk the runs of the 16-bit equality mask
        uint32_t r = t.run, pos = 0;
        const uint32_t nvp = t.nvp;
        if (t.eqm | r) {
            while (pos < nvp) {
                const uint32_t m = t.eqm >> pos;
                const uint32_t ones = min((uint32_t)__ffs((int)~m) - 1u, nvp - pos);     // leading equal pixels
                if (ones) {
                    r += ones; pos += ones;
                    if (r >= M) { bits += s_match[M]; r -= M; }
                    if (pos >= nvp) break;
                }
                if (r) { bits += run_bits16<LIT1>(s_lit, s_match, r, px, left, pos); r = 0; }   // a literal follows: flush the remainder
                const uint32_t mz = t.eqm >> pos;
                const uint32_t zeros = mz ? (uint32_t)__ffs((int)mz) - 1u : 32u;
                pos += zeros;
            }
        }
        if (t.last) {
            if (r) bits += run_bits16<LIT1>(s_lit, s_match, r, px, left, nvp);
            // capacity rule (SURVEY Q5): size of the scanline's last flush unit
            const uint32_t k = nvp - 1u;
            if (t.litm & (1u << k)) {
                uint32_t lastpx = px[0];
#pragma unroll
                for (int q = 1; q < 16; q++) lastpx = (k == (uint32_t)q) ? px[q] : lastpx;
                last_unit = literal_bits16<CHANS>(s_lit, lastpx) + ((w == 1 && p.merge_first_unit) ? s_lit[filt] : 0u);
            } else last_unit = r ? s_match[r] : s_match[M];
            if constexpr (LIT1) if (r == 1u && !(t.litm & (1u << k))) last_unit = run_bits16<true>(s_lit, s_match, r, px, left, nvp);
            if (y == p.h - 1) p.st[img].last_unit_bits = last_unit;
        }
        // bit offset of this lane's first token inside the row (the pack kernel starts writing there)
        uint32_t step_bits;
        const uint32_t ex = warp_excl_scan_u32(bits, lane, step_bits);
        lane_ofs[step * 32u + lane] = make_uint2(row_run + ex, lane_info16(t));     // the pack kernel starts from these instead of re-classifying
        row_run += step_bits;
    }

    const unsigned long long A = warp_sum_u64(sumA);
    const unsigned long long B = warp_sum_u64(sumB);
    if (lane == 0) {
        const unsigned long long n = (unsigned long long)bpl + 1ull;
        const unsigned long long S1 = A + filt;
        const unsigned long long S2 = n * S1 - (A + B);
        p.row_bits[(size_t)img * p.h + y] = row_run;
        p.row_adler[(size_t)img * p.h + y] = make_uint2((uint32_t)(S1 % kAdlerMod), (uint32_t)(S2 % kAdlerMod));
    }
}

// ------------------------------------------------------------------------------------------------
// K1-hist (v2): 288-bin literal/length histogram of 2-pass mode (fpng.cpp:1021-1084, 1299-1363) on the 16-pixel walker.
// Warp-private shared-memory histograms (no inter-warp contention), merged per CTA, then added to the image's bins.
// ------------------------------------------------------------------------------------------------
template <int CHANS, int LOAD, bool RAGGED = false>
__global__ void __launch_bounds__(32 * kScan16Rows) row_hist16_kernel(std::conditional_t<RAGGED, RaggedParams<ScanParams>, ScanParams> p)
{
    using WK = typename Loader16<CHANS, LOAD>::type;
    constexpr uint32_t M = max_match_pixels(CHANS);
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    uint32_t* s_hist_all = reinterpret_cast<uint32_t*>(dyn_smem + kScan16Rows * WK::kWarpBytes);   // [warps][288]
    __shared__ uint16_t s_lensym[88];

    const uint32_t lane = threadIdx.x & 31, warp = __shfl_sync(kFullMask, threadIdx.x >> 5, 0);   // warp-uniform for the compiler (see the scan kernel)
    uint32_t img = blockIdx.y, cta = blockIdx.x;
    if constexpr (RAGGED) { p.hist += (size_t)ragged_image16(p, cta) * 288; img = 0; }
    const uint32_t y = cta * kScan16Rows + warp;
    for (uint32_t i = threadIdx.x; i < kScan16Rows * 288; i += blockDim.x) s_hist_all[i] = 0u;
    if (threadIdx.x >= 1 && threadIdx.x <= M) { uint32_t sy, xb, xv; deflate_len_code(threadIdx.x * CHANS, sy, xb, xv); s_lensym[threadIdx.x] = (uint16_t)sy; }
    __syncthreads();
    uint32_t* hist = s_hist_all + warp * 288;

    if (y < p.h) {
        const uint32_t w = p.w, bpl = w * CHANS;
        const uint8_t* cur = p.pixels + (size_t)img * p.image_stride + (size_t)y * p.row_pitch;
        const uint8_t* prev = y ? cur - p.row_pitch : nullptr;
        const uint32_t nsteps = (w + kStep16 - 1) / kStep16;
        uint8_t* tiles = dyn_smem + warp * WK::kWarpBytes;
        WK wk; wk.init(lane, tiles); wk.bind(cur, prev); set_planes(wk, p.chan_stride);
        RowCarry carry = {0u, 0u};
        uint32_t dummyA = 0; unsigned long long dummyB = 0;
        if (lane == 0) atomicAdd(&hist[y ? 2 : 0], 1u);               // the filter literal
        wk.prefetch(cur, prev, 0, bpl, lane, tiles);
        for (uint32_t step = 0; step < nsteps; step++) {
            uint32_t dw[WK::kWords], px[16];
            wk.template consume<false>(prev != nullptr, step, step, bpl, lane, tiles, dw, dummyA, dummyB);
            if (step + 1 < nsteps) wk.prefetch(cur, prev, step + 1, bpl, lane, tiles);
            WK::pixels(dw, px);
            const uint32_t p0 = step * kStep16 + lane * kPix16;
            const Lane16 t = classify16<CHANS>(px, p0, w, carry, lane);
            if (__any_sync(kFullMask, t.litm != 0)) {
#pragma unroll
                for (int k = 0; k < 16; k++) {
                    if (t.litm & (1u << k)) {
                        atomicAdd(&hist[px[k] & 0xFFu], 1u);
                        atomicAdd(&hist[byte1(px[k])], 1u);
                        if (CHANS == 4) { atomicAdd(&hist[byte2(px[k])], 1u); atomicAdd(&hist[px[k] >> 24], 1u); }
                        else atomicAdd(&hist[px[k] >> 16], 1u);
                    }
                }
            }
            uint32_t r = t.run, pos = 0;
            const uint32_t nvp = t.nvp;
            if (t.eqm | r) {
                while (pos < nvp) {
                    const uint32_t m = t.eqm >> pos;
                    const uint32_t ones = min((uint32_t)__ffs((int)~m) - 1u, nvp - pos);
                    if (ones) {
                        r += ones; pos += ones;
                        if (r >= M) { atomicAdd(&hist[s_lensym[M]], 1u); r -= M; }
                        if (pos >= nvp) break;
                    }
                    if (r) { atomicAdd(&hist[s_lensym[r]], 1u); r = 0; }
                    const uint32_t mz = t.eqm >> pos;
                    pos += mz ? (uint32_t)__ffs((int)mz) - 1u : 32u;
                }
            }
            if (t.last && r) atomicAdd(&hist[s_lensym[r]], 1u);
        }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < 288; i += blockDim.x) {
        uint32_t v = 0;
#pragma unroll
        for (int wq = 0; wq < kScan16Rows; wq++) v += s_hist_all[wq * 288 + i];
        if (v) atomicAdd(&p.hist[(size_t)img * 288 + i], v);
    }
}

// ------------------------------------------------------------------------------------------------
// K3 (v2): pack.  Every lane knows where its 16 pixels' tokens start and how they classify (lane_ofs from the scan
// kernel: bit offset + lane_info16), so it emits its codes through a 32-bit accumulator straight into the warp's staging
// words.  A staging word is COMPLETED (its bit 31 written) by exactly one lane, which stores it with a plain store; the
// bits other lanes own in that word (their last, partial word) are OR-ed in after a warp barrier.  Nothing is re-zeroed
// between steps except the one word no lane completes (the step's last, partial word), and lane 0 carries that word's
// bits into the next step in a register.
// ------------------------------------------------------------------------------------------------
// 32-bit shared-window addresses keep the stager's running pointer in ONE register (with a generic pointer the compiler
// carried two copies and incremented both on every put)
__device__ __forceinline__ void sts_u32(uint32_t saddr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;\n" :: "r"(saddr), "r"(v)); }
__device__ __forceinline__ void reds_or_u32(uint32_t saddr, uint32_t v) { asm volatile("red.shared.or.b32 [%0], %1;\n" :: "r"(saddr), "r"(v)); }
__device__ __forceinline__ uint32_t lds_u32(uint32_t saddr) { uint32_t v; asm("ld.shared.u32 %0, [%1];\n" : "=r"(v) : "r"(saddr)); return v; }

struct BitStager16 {
    uint32_t cur, n;            // word being filled (n < 32 valid bits)
    uint32_t dst;               // shared-memory address of the staging word `cur` goes to
    __device__ __forceinline__ void begin(uint32_t stage_saddr, uint32_t bitpos, uint32_t seed)
    {
        cur = seed; n = bitpos & 31u; dst = stage_saddr + ((bitpos >> 5) << 2);
    }
    // append `len` (<= 32, code < 2^len) bits; len == 0 (code == 0) is a no-op
    __device__ __forceinline__ void put(uint32_t code, uint32_t len)
    {
        const uint32_t lo = cur | (code << n);
        const uint32_t hi = __funnelshift_l(code, 0u, n);               // bits that spill into the next word (0 when n == 0)
        const uint32_t n2 = n + len;
        if (n2 >= 32u) { sts_u32(dst, lo); dst += 4u; cur = hi; } else cur = lo;   // this lane owns bit 31 of the word: plain store
        n = n2 & 31u;
    }
    // after a warp barrier: the partial last word is shared with the next lane's first word
    __device__ __forceinline__ void end() { if (cur) reds_or_u32(dst, cur); }
};

__device__ __forceinline__ void put_pair16(BitStager16& bs, uint32_t a, uint32_t b)   // two table entries (len << 16 | code), <= 24 bits
{
    const uint32_t la = a >> 16;
    bs.put((a & 0xFFFFu) | ((b & 0xFFFFu) << la), la + (b >> 16));
}
__device__ __forceinline__ void put_match16(BitStager16& bs, uint32_t s_match_saddr, uint32_t r)
{
    const uint32_t m = lds_u32(s_match_saddr + r * 4u);
    bs.put(m & 0xFFFFFFu, m >> 24);
}

// Literal codes come as (code, size) register pairs from one 64-bit shared load per byte, instead of a packed 32-bit entry whose
// fields have to be shifted / masked apart (2 ALU instructions less per literal; the pack kernel is ALU-pipe bound).  The 8-byte
// table [512][2] sits directly below the 4-byte one in shared memory; its upper half is all zero: a "null" entry of 0 bits, which
// switches a pixel's literals off without a branch.
__device__ __forceinline__ uint2 lds_u64(uint32_t saddr) { uint2 v; asm("ld.shared.v2.u32 {%0, %1}, [%2];\n" : "=r"(v.x), "=r"(v.y) : "r"(saddr)); return v; }
template <int POS>
__device__ __forceinline__ uint32_t lit_off16x8(uint32_t w, uint32_t nb8)
{
    const uint32_t x = POS == 0 ? (w << 3) : (POS == 1 ? (w >> 5) : (POS == 2 ? (w >> 13) : (w >> 21)));
    return (x & 0x7F8u) | nb8;
}
// the all-literal path's offset: "extract the byte (one ALU-pipe instruction), multiply by 8 (IMAD with a constant-bank operand,
// FMA pipe)" instead of shift + mask (two ALU-pipe instructions).  Measured on an H100 (700 W) as fast as shift + mask (C2 pack
// 1.636-1.646 against 1.642 ms); kept for its lower ALU-pipe count.
template <int POS>
__device__ __forceinline__ uint32_t lit_off16x8_plain(uint32_t w)
{
    const uint32_t b = POS == 0 ? (w & 0xFFu) : (POS == 1 ? byte1(w) : (POS == 2 ? byte2(w) : (w >> 24)));
    return b * c_fma_k[5];
}

// byte offset of the packed 32-bit (size << 16 | code) entry of byte POS of word w
template <int POS>
__device__ __forceinline__ uint32_t lit_off16(uint32_t w)
{
    const uint32_t x = POS == 0 ? (w << 2) : (POS == 1 ? (w >> 6) : (POS == 2 ? (w >> 14) : (w >> 22)));
    return x & 0x3FCu;
}

template <int CHANS>
__device__ __forceinline__ void put_literal16(BitStager16& bs, uint32_t s_lit_saddr, uint32_t px)
{
    put_pair16(bs, lds_u32(s_lit_saddr + lit_off16<0>(px)), lds_u32(s_lit_saddr + lit_off16<1>(px)));
    if (CHANS == 4) put_pair16(bs, lds_u32(s_lit_saddr + lit_off16<2>(px)), lds_u32(s_lit_saddr + lit_off16<3>(px)));
    else { const uint32_t c2 = lds_u32(s_lit_saddr + lit_off16<2>(px)); bs.put(c2 & 0xFFFFu, c2 >> 16); }
}

// the 4 literal codes of one 32-bit word of filtered bytes, in byte order, as two <= 24-bit puts (the all-literal path)
__device__ __forceinline__ void put_word16(BitStager16& bs, uint32_t s_lit_saddr, uint32_t w)
{
    const uint32_t l64 = s_lit_saddr - 4096u;
    const uint2 f0 = lds_u64(l64 + lit_off16x8_plain<0>(w)), f1 = lds_u64(l64 + lit_off16x8_plain<1>(w));
    const uint2 f2 = lds_u64(l64 + lit_off16x8_plain<2>(w)), f3 = lds_u64(l64 + lit_off16x8_plain<3>(w));
    bs.put(f0.x | (f1.x << f0.y), f0.y + f1.y);
    bs.put(f2.x | (f3.x << f2.y), f2.y + f3.y);
}

// pending run length before pixel kk (0..16) of a lane, from its equality mask and the run entering the lane
template <uint32_t M>
__device__ __forceinline__ uint32_t run_before16(uint32_t eqm, uint32_t r_in, uint32_t kk)
{
    const uint32_t t = ~eqm & ((1u << kk) - 1u);                         // non-match pixels below kk
    if (t == 0u) { const uint32_t r = kk + r_in; return r >= M ? r - M : r; }
    return kk - 1u - (31u - (uint32_t)__clz((int)t));
}

// a pending run of r > 0 pixels whose last pixel is `covered`.  LIT1: a one-pixel match is written as that pixel's four literals
// when the match costs more bits (fpng.cpp:1520-1528; the scan kernel counted the same choice)
template <bool LIT1>
__device__ __forceinline__ void put_run16(BitStager16& bs, uint32_t s_lit_saddr, uint32_t s_match_saddr, uint32_t r, uint32_t covered)
{
    if (LIT1 && r == 1u) {
        const uint32_t c0 = lds_u32(s_lit_saddr + lit_off16<0>(covered)), c1 = lds_u32(s_lit_saddr + lit_off16<1>(covered));
        const uint32_t c2 = lds_u32(s_lit_saddr + lit_off16<2>(covered)), c3 = lds_u32(s_lit_saddr + lit_off16<3>(covered));
        const uint32_t m = lds_u32(s_match_saddr + 4u);
        if ((m >> 24) > (c0 >> 16) + (c1 >> 16) + (c2 >> 16) + (c3 >> 16)) { put_pair16(bs, c0, c1); put_pair16(bs, c2, c3); return; }
    }
    put_match16(bs, s_match_saddr, r);
}

// a token event at pixel kk: the run reaches M at this (match) pixel, or a pending run is flushed before this literal
// (LIT1: `covered` is pixel kk - 1, see put_run16)
template <uint32_t M, bool LIT1 = false>
__device__ __forceinline__ void put_event16(BitStager16& bs, uint32_t s_match_saddr, uint32_t eqm, uint32_t r_in, uint32_t kk,
                                            uint32_t s_lit_saddr = 0u, uint32_t covered = 0u)
{
    const uint32_t len = ((eqm >> kk) & 1u) ? M : run_before16<M>(eqm, r_in, kk);
    if (len) put_run16<LIT1>(bs, s_lit_saddr, s_match_saddr, len, covered);
}

// the literal codes of word J (0 .. kHalfWords-1) of a mixed half: one 64-bit (code, size) load per byte, each byte's entry taken
// from the table's null half when its pixel is not a literal, two codes per put.  A token event goes before its pixel's first byte:
// for RGB that byte can sit inside the word, and only then (rare: a run ends or reaches M in this word) the word is put code by
// code with the match token in between.
__device__ __forceinline__ uint32_t null_ofs8(uint32_t nl, int k) { return (nl << (11 - k)) & 0x800u; }   // bit k of nl -> 0x800 (k <= 7)
// LIT1 (RGBA, one pixel per word): prev is the pixel before the word's
template <int CHANS, int J, uint32_t M, bool LIT1>
__device__ __forceinline__ void put_mixed_word16(BitStager16& bs, uint32_t lit_s, uint32_t match_s, uint32_t w, uint32_t nl, uint32_t ev8,
                                                 uint32_t eqm, uint32_t r_in, uint32_t kbase, uint32_t prev)
{
    constexpr int kFirst = 4 * J / CHANS;                              // pixel of byte 0
    constexpr int kIn = (4 * J + 3) / CHANS;                           // pixel of byte 3: starts inside the word iff kIn != kFirst (RGB)
    constexpr int kSplit = CHANS * kIn - 4 * J;                        // its first byte (1..3)
    const uint32_t l64 = lit_s - 4096u;
    const uint2 f0 = lds_u64(l64 + lit_off16x8<0>(w, null_ofs8(nl, kFirst)));
    const uint2 f1 = lds_u64(l64 + lit_off16x8<1>(w, null_ofs8(nl, (4 * J + 1) / CHANS)));
    const uint2 f2 = lds_u64(l64 + lit_off16x8<2>(w, null_ofs8(nl, (4 * J + 2) / CHANS)));
    const uint2 f3 = lds_u64(l64 + lit_off16x8<3>(w, null_ofs8(nl, kIn)));
    if (CHANS * kFirst == 4 * J && (ev8 & (1u << kFirst))) put_event16<M, LIT1>(bs, match_s, eqm, r_in, kbase + kFirst, lit_s, prev);
    if (kIn != kFirst && (ev8 & (1u << kIn))) {
        const uint2 f[4] = {f0, f1, f2, f3};
#pragma unroll
        for (int b = 0; b < 4; b++) {
            if (b == kSplit) put_event16<M>(bs, match_s, eqm, r_in, kbase + kIn);
            bs.put(f[b].x, f[b].y);
        }
        return;
    }
    bs.put(f0.x | (f1.x << f0.y), f0.y + f1.y);
    bs.put(f2.x | (f3.x << f2.y), f2.y + f3.y);
}
// words J.. of a mixed half (hw: its 2 * CHANS filtered words; nl: bit k set when pixel k is not a literal; before: LIT1, the pixel
// before the half)
template <int CHANS, uint32_t M, bool LIT1, int J = 0>
__device__ __forceinline__ void put_mixed_half16(BitStager16& bs, uint32_t lit_s, uint32_t match_s, const uint32_t (&hw)[2 * CHANS], uint32_t nl,
                                                 uint32_t ev8, uint32_t eqm, uint32_t r_in, uint32_t kbase, uint32_t before)
{
    put_mixed_word16<CHANS, J, M, LIT1>(bs, lit_s, match_s, hw[J], nl, ev8, eqm, r_in, kbase, J ? hw[J ? J - 1 : 0] : before);
    if constexpr (J + 1 < 2 * CHANS) put_mixed_half16<CHANS, M, LIT1, J + 1>(bs, lit_s, match_s, hw, nl, ev8, eqm, r_in, kbase, before);
}

// one Horner step of the in-kernel CRC: the register (XOR-ed with the lane's previous word) advanced over 128 bytes, then the next
// word (slice tables [4][256] at shared address crc_s; byte extraction with PRMT so that each look-up address is one LEA).
// Nibble tables [8][16] (every look-up conflict free: 1 instead of ~3 wavefronts) measured slower: the 8 extra ALU instructions
// per word cost more than the bank conflicts (DESIGN 4.1).
__device__ __forceinline__ uint32_t crc_step16(uint32_t crc_s, uint32_t cx, uint32_t v)
{
    const uint32_t b0 = cx & 0xFFu, b1 = __byte_perm(cx, 0u, 0x4441), b2 = __byte_perm(cx, 0u, 0x4442), b3 = cx >> 24;
    return v ^ lds_u32(crc_s + b0 * 4u) ^ lds_u32(crc_s + 1024u + b1 * 4u) ^ lds_u32(crc_s + 2048u + b2 * 4u) ^ lds_u32(crc_s + 3072u + b3 * 4u);
}

template <int CHANS, int LOAD, bool RAGGED = false, bool LIT1 = false>
__global__ void __launch_bounds__(32 * pack16_warps(CHANS)) pack_rows16_kernel(std::conditional_t<RAGGED, RaggedParams<PackParams>, PackParams> p,
                                                                       uint32_t rows_per_warp)
{
    static_assert(!LIT1 || CHANS == 4, "the one-pixel-match rule is RGBA only");
    using WK = typename Loader16<CHANS, LOAD>::type;
    uint32_t img = blockIdx.y, cta = blockIdx.x;
    if constexpr (RAGGED) {
        const ImageDesc& d = p.ragged.desc[ragged_image16(p, cta)];
        p.row_ofs += d.row_base; p.row_crc += d.row_base; p.out += d.out_ofs; p.out_stride = 0;
        img = 0;
    }
    if (p.stored_only && !p.st[img].stored) return;     // after the fused encoder only stored-block images are left to write
    constexpr uint32_t M = max_match_pixels(CHANS);
    constexpr int kHalfWords = 2 * CHANS;        // filtered words of 8 pixels
    constexpr int kPack16Rows = pack16_warps(CHANS);
    extern __shared__ __align__(16) uint8_t dyn_smem[];
    uint32_t* s_lit64 = reinterpret_cast<uint32_t*>(dyn_smem + kPack16Rows * WK::kWarpBytes);   // [512][2]: (code, size) + null half
    uint32_t* s_lit = s_lit64 + 1024;                // [256]: packed entries (size << 16 | code)
    uint32_t* s_match = s_lit + 256;
    uint32_t* s_stage_all = s_match + 88;
    uint32_t* s_crc = s_stage_all + kPack16Rows * stage16_words<CHANS>();              // [4][256] CRC slice tables (row_crc only)

    const uint32_t lane = threadIdx.x & 31, warp = __shfl_sync(kFullMask, threadIdx.x >> 5, 0);   // warp-uniform for the compiler (see the scan kernel)
    const uint32_t row0 = (cta * kPack16Rows + warp) * rows_per_warp;                  // this warp's first scanline
    const bool do_crc = p.row_crc != nullptr;
    const CodeBook* book = p.books + (size_t)img * p.book_stride;
    const ImageState st = p.st[img];
    if (st.stored) {                             // stored-block fallback (fpng.cpp:818-866): strided copy of the rows
        const uint32_t bpl_s = p.w * CHANS;
        for (uint32_t y = row0; y < min(row0 + rows_per_warp, p.h); y++) {
            const uint8_t* row = p.pixels + (size_t)img * p.image_stride + (size_t)y * p.row_pitch;
            uint8_t* zl = p.out + (size_t)img * p.out_stride + kPngHeaderSize;
            if (LOAD == kLoad16Planar) store_row_raw(PlaneBytes<CHANS>{row, p.chan_stride}, zl, y, bpl_s, lane, &p.row_adler[(size_t)img * p.h + y]);
            else store_row_raw(row, zl, y, bpl_s, lane, &p.row_adler[(size_t)img * p.h + y]);
        }
        return;
    }
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) {
        const uint32_t e = book->lit[i];
        s_lit[i] = e;
        s_lit64[2 * i] = e & 0xFFFFu; s_lit64[2 * i + 1] = e >> 16; s_lit64[512 + 2 * i] = 0u; s_lit64[512 + 2 * i + 1] = 0u;
    }
    if (threadIdx.x < 88) s_match[threadIdx.x] = book->match[threadIdx.x];
    if (do_crc) for (uint32_t i = threadIdx.x; i < 1024; i += blockDim.x) s_crc[i] = __ldg(p.crc_f128b + i);
    __syncthreads();
    if (row0 >= p.h) return;

    const uint32_t w = p.w, bpl = w * CHANS;
    const uint32_t nrows = min(rows_per_warp, p.h - row0);
    const uint32_t crc_s = smem_u32(s_crc);
    // CRC of the scanline's code words (PackParams::row_crc): lane l owns the words whose index in the scanline is l (mod 32),
    // a Horner recurrence over 128-byte strides; cx is the register XOR-ed with the lane's latest word, not yet advanced
    uint32_t cx = 0;
    const uint8_t* img_px = p.pixels + (size_t)img * p.image_stride;
    uint32_t* stage = s_stage_all + warp * stage16_words<CHANS>();
    const uint32_t stage_s = smem_u32(stage), lit_s = smem_u32(s_lit), match_s = smem_u32(s_match);
    uint8_t* tiles = dyn_smem + warp * WK::kWarpBytes;
    const uint32_t nsteps = (w + kStep16 - 1) / kStep16;
    const uint32_t nitems = nrows * nsteps;      // (scanline, step) work items of this warp, walked as one pipelined sequence
    // per-row constants of all this warp's rows, one row per lane (broadcast at the row's first step)
    const size_t ridx0 = (size_t)img * p.h + row0;
    const unsigned long long my_G = lane < nrows ? p.row_ofs[ridx0 + lane] : 0ull;
    const uint32_t my_total = lane < nrows ? p.row_bits[ridx0 + lane] : 0u;
    const uint2* lane_ofs = p.lane_ofs + ridx0 * p.lane_ofs_pitch + lane;              // this lane's entry of (row0, step 0)

    uint32_t* gptr = nullptr;                    // global word that stage[0] maps to; advanced as words are flushed
    bool first_pending = true;                   // the row's first word is shared with the previous row / the block header
    uint32_t g31 = 0, row_total = 0;
    uint32_t flushed_bits = 0;                   // row bits (incl. the G & 31 lead-in) already flushed to global, multiple of 32
    uint32_t leftover = 0;                       // bits of the partially filled word carried from the previous step (lane 0 seeds with it)
    // LIT1: lane 31's last pixel of the previous step.  Not reset at a scanline's start: no run enters its first lane, so it is unread there
    uint32_t prev_px = 0;

    WK wk; wk.init(lane, tiles); set_planes(wk, p.chan_stride);
    uint32_t dummyA = 0; unsigned long long dummyB = 0;
    const uint32_t pitch = p.row_pitch;
    // the current item's scanline, advanced by the pitch at each row end (recomputing img_px + y * pitch per item costs the RGBA
    // direct-loader kernel 9 registers)
    const uint8_t* row_px = img_px + (size_t)row0 * pitch;
    wk.prefetch(row_px, row0 ? row_px - pitch : nullptr, 0, bpl, lane, tiles);
    uint2 mine = lane_ofs[0];
    uint32_t r_i = 0, step = 0;                  // row (relative to row0) and step of the current item
    for (uint32_t item = 0; item < nitems; item++) {
        const uint32_t y = row0 + r_i;
        if (step == 0) {
            const unsigned long long G = __shfl_sync(kFullMask, my_G, r_i);
            row_total = __shfl_sync(kFullMask, my_total, r_i);
            gptr = reinterpret_cast<uint32_t*>(p.out + (size_t)img * p.out_stride) + (G >> 5);
            g31 = (uint32_t)(G & 31ull);
            first_pending = true; flushed_bits = 0; leftover = 0;
        }
        uint32_t dw[WK::kWords];
        wk.bind(row_px, y ? row_px - pitch : nullptr);
        wk.template consume<false>(y != 0, item, step, bpl, lane, tiles, dw, dummyA, dummyB);
        // the next item (possibly the first step of the next scanline) is fetched while this one is emitted
        const bool more = step + 1 < nsteps;     // more steps in this row
        const uint32_t my_ofs = mine.x, info = mine.y;
        if (item + 1 < nitems) {
            const uint32_t ny = more ? y : y + 1, nstep = more ? step + 1 : 0;
            const uint8_t* nc = img_px + (size_t)ny * pitch;
            wk.prefetch(nc, ny ? nc - pitch : nullptr, nstep, bpl, lane, tiles);
            mine = lane_ofs[(size_t)(ny - row0) * p.lane_ofs_pitch + nstep * 32u];
        }
        // classification of this lane's 16 pixels, as computed by the scan kernel
        const uint32_t eqm = info & 0xFFFFu, r_in = (info >> 16) & 0x7Fu, nvp = (info >> 23) & 0x1Fu;
        const uint32_t litm = ((1u << nvp) - 1u) & ~eqm;
        // token events: a pending run flushed before a literal pixel, or the run reaching M at a match pixel (at most one per lane)
        const uint32_t lead = (uint32_t)__ffs((int)~eqm) - 1u;          // leading match pixels (<= 16)
        const uint32_t kM = M - 1u - r_in;
        const uint32_t evm = (litm & ((eqm << 1) | (r_in ? 1u : 0u))) | (kM < lead ? (1u << kM) : 0u);

        BitStager16 bs;
        // staging bit 0 corresponds to row bit (flushed_bits - g31); the filter literal sits at row bit 0
        if (lane == 0) {
            if (step == 0) { const uint32_t fcode = s_lit[y ? 2 : 0]; bs.begin(stage_s, g31, 0u); bs.put(fcode & 0xFFFFu, fcode >> 16); }
            else bs.begin(stage_s, g31 + my_ofs - flushed_bits, leftover);
        } else bs.begin(stage_s, g31 + my_ofs - flushed_bits, 0u);
        // The 16 pixels are emitted as 2 halves of 8 by a ROLLED loop (a fully unrolled body is ~80 KB of SASS and stalls
        // on instruction fetch: ncu no_instruction dominated).  Per half one of four warp-uniform paths:
#pragma unroll 1
        for (uint32_t h = 0; h < 2; h++) {
            const uint32_t lit8 = (litm >> (8u * h)) & 0xFFu, ev8 = (evm >> (8u * h)) & 0xFFu;
            uint32_t hw[kHalfWords];
#pragma unroll
            for (int j = 0; j < kHalfWords; j++) hw[j] = h ? dw[kHalfWords + j] : dw[j];
            uint32_t before = 0;                 // LIT1: the pixel before the half, which a run entering it covers
            if constexpr (LIT1) {
                const uint32_t up = __shfl_up_sync(kFullMask, dw[15], 1);
                before = h ? dw[kHalfWords - 1] : (lane ? up : prev_px);
            }
            if (__all_sync(kFullMask, lit8 == 0xFFu && ev8 == 0u)) {
                // (1) all 256 pixels are literals, no run pending (noisy rows): the filtered bytes in order, two codes per put
#pragma unroll
                for (int j = 0; j < kHalfWords; j++) put_word16(bs, lit_s, hw[j]);
            } else if (__all_sync(kFullMask, lit8 == 0u)) {
                // (2) no literal at all (inside long runs): only a run reaching M emits a token
                if (ev8) put_match16(bs, match_s, M);
            } else if (__reduce_add_sync(kFullMask, (uint32_t)__popc(lit8)) >= 16u) {
                // (3) mixed: the all-literal emission word by word, each byte switched off through the table's null half when
                //     its pixel is not a literal; the rare run tokens are inserted by a per-word event check
                put_mixed_half16<CHANS, M, LIT1>(bs, lit_s, match_s, hw, ~lit8, ev8, eqm, r_in, 8u * h, before);
            } else {
                // (4) sparse literals (RLE-dominated rows): per-pixel token walk, 4 pixels at a time
                uint32_t r = run_before16<M>(eqm, r_in, 8u * h);
#pragma unroll 1
                for (uint32_t g = 0; g < 2; g++) {
                    uint32_t q[4];
                    if (CHANS == 4) {
#pragma unroll
                        for (int j = 0; j < 4; j++) q[j] = g ? hw[4 + j] : hw[j];
                    } else {
                        const uint32_t w0 = g ? hw[3] : hw[0], w1 = g ? hw[4] : hw[1], w2 = g ? hw[5] : hw[2];
                        q[0] = w0 & 0x00FFFFFFu;
                        q[1] = __byte_perm(w0, w1, 0x4543) & 0x00FFFFFFu;
                        q[2] = __byte_perm(w1, w2, 0x4432) & 0x00FFFFFFu;
                        q[3] = w2 >> 8;
                    }
                    const uint32_t e4 = eqm >> (8u * h + 4u * g), base = 8u * h + 4u * g;
                    const uint32_t pb = g ? hw[3] : before;                                   // LIT1: the pixel before q[0]
#pragma unroll
                    for (int j = 0; j < 4; j++) {
                        if (base + j < nvp) {
                            if (e4 & (1u << j)) {
                                if (++r == M) { put_match16(bs, match_s, M); r = 0; }
                            } else {
                                if (r) { put_run16<LIT1>(bs, lit_s, match_s, r, j ? q[j ? j - 1 : 0] : pb); r = 0; }
                                put_literal16<CHANS>(bs, lit_s, q[j]);
                            }
                        }
                    }
                }
            }
        }
        if constexpr (LIT1) prev_px = __shfl_sync(kFullMask, dw[15], 31);
        if (info >> 28) {                                                // this lane holds the scanline's last pixel: flush the trailing run
            const uint32_t r = run_before16<M>(eqm, r_in, nvp);
            if (r) put_run16<LIT1>(bs, lit_s, match_s, r, pixel_before16(dw, 0u, nvp));   // nvp >= 1
        }
        // row bits after this step (the next step's first offset was loaded a whole emission ago)
        const uint32_t step_end = more ? __shfl_sync(kFullMask, mine.x, 0) : row_total;
        const uint32_t fill = g31 + step_end - flushed_bits;            // live bits in the staging buffer after this step
        const uint32_t nwords = fill >> 5;
        if (lane == 0) stage[nwords] = 0u;                               // the one word no lane completes in this step
        __syncwarp();                                                    // all complete words are stored ...
        bs.end();                                                        // ... before the partial ones are OR-ed in
        __syncwarp();

        // ---- flush the complete words; carry the partial one in a register
        leftover = stage[nwords];
        // lanes take the words in scanline order rotated by the words already flushed, so that a lane always sees stride 32
        {
            uint32_t j = (lane - (flushed_bits >> 5)) & 31u;
            const uint32_t* sp = stage + j;
            uint32_t* gp = gptr + j;
            if (first_pending && j == 0u && nwords) {                    // the scanline's first word is shared with its predecessor
                const uint32_t v = *sp;
                atomicOr(gp, v);
                if (do_crc) cx = crc_step16(crc_s, cx, v);
                j = 32u; sp += 32; gp += 32;
            }
            for (; j < nwords; j += 32u, sp += 32, gp += 32) {
                const uint32_t v = *sp;
                *gp = v;
                if (do_crc) cx = crc_step16(crc_s, cx, v);
            }
        }
        __syncwarp();                                                    // staging is rewritten by the next step
        if (nwords) first_pending = false;
        gptr += nwords;
        flushed_bits += nwords << 5;
        if (more) step++;
        else {                                                           // end of the scanline: its last, partial word
            if (lane == 0 && leftover) atomicOr(gptr, leftover);
            if (do_crc) {
                // the partial word (possibly empty) counts as word Wn; every lane's value is shifted to the end of word Wn
                const uint32_t Wn = flushed_bits >> 5;
                if (lane == (Wn & 31u)) cx = crc_step16(crc_s, cx, leftover);
                const uint32_t* lm = p.crc_lane_mul + (31u - ((Wn - lane) & 31u)) * 128u;    // x^(32 * (words after the lane's last + 1))
                uint32_t r = __ldg(lm + (cx & 15u));
#pragma unroll
                for (int t = 1; t < 8; t++) r ^= __ldg(lm + 16 * t + ((cx >> (4 * t)) & 15u));
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) r ^= __shfl_xor_sync(kFullMask, r, o);
                if (lane == 0) p.row_crc[ridx0 + r_i] = r;
                cx = 0;
            }
            step = 0; r_i++; row_px += pitch;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
bool walk16_eligible(const void* base, size_t image_stride, uint32_t row_pitch, uint32_t w, uint32_t chans)
{
    const size_t bpl = (size_t)w * chans;
    return ((uintptr_t)base % 16 == 0) && (image_stride % 16 == 0) && (row_pitch % 16 == 0) && (bpl % 16 == 0);
}
template <class P> static int load16_mode(const P& p, uint32_t chans)
{
    if (p.chan_stride) return kLoad16Planar;
    return walk16_eligible(p.pixels, p.image_stride, p.row_pitch, p.w, chans) ? kLoad16Staged : kLoad16Direct;
}

template <int CHANS, int LOAD> constexpr size_t scan16_smem() { return kScan16Rows * Loader16<CHANS, LOAD>::type::kWarpBytes + 256 + 96; }
template <int CHANS, int LOAD> constexpr size_t pack16_smem()
{
    return pack16_warps(CHANS) * Loader16<CHANS, LOAD>::type::kWarpBytes + (1024 + 256 + 88 + pack16_warps(CHANS) * stage16_words<CHANS>() + 1024) * 4;
}
template <int CHANS, int LOAD> constexpr size_t hist16_smem() { return kScan16Rows * Loader16<CHANS, LOAD>::type::kWarpBytes + kScan16Rows * 288 * 4; }

// The 16-pixel kernels take any scanline alignment and either layout: `load` (load16_mode()) selects the loader.
// R: the ragged instantiation (the uniform launches pass false)
#define FPNGB_LAUNCH16_ONE(C, L, R, kernel, smemfn, grid, threads, ...) do { \
        FPNGB_SET_SMEM((kernel<C, L, R>), (smemfn<C, L>())); kernel<C, L, R><<<grid, threads, smemfn<C, L>(), s>>>(__VA_ARGS__); } while (0)
#define FPNGB_LAUNCH16(kernel, R, smemfn, grid, threads, ...) do { \
        if (chans == 4) { \
            if (load == kLoad16Planar) FPNGB_LAUNCH16_ONE(4, kLoad16Planar, R, kernel, smemfn, grid, threads, __VA_ARGS__); \
            else if (load == kLoad16Direct) FPNGB_LAUNCH16_ONE(4, kLoad16Direct, R, kernel, smemfn, grid, threads, __VA_ARGS__); \
            else FPNGB_LAUNCH16_ONE(4, kLoad16Staged, R, kernel, smemfn, grid, threads, __VA_ARGS__); \
        } else { \
            if (load == kLoad16Planar) FPNGB_LAUNCH16_ONE(3, kLoad16Planar, R, kernel, smemfn, grid, threads, __VA_ARGS__); \
            else if (load == kLoad16Direct) FPNGB_LAUNCH16_ONE(3, kLoad16Direct, R, kernel, smemfn, grid, threads, __VA_ARGS__); \
            else FPNGB_LAUNCH16_ONE(3, kLoad16Staged, R, kernel, smemfn, grid, threads, __VA_ARGS__); \
        } \
    } while (0)
// the RGBA scan and pack kernels with the one-pixel-match rule (ScanParams / PackParams::lit1_rule)
#define FPNGB_TARGS(...) __VA_ARGS__
#define FPNGB_LAUNCH16_LIT1(kernel, R, smemfn, grid, threads, ...) do { \
        if (load == kLoad16Planar) FPNGB_LAUNCH16_ONE(4, kLoad16Planar, FPNGB_TARGS(R, true), kernel, smemfn, grid, threads, __VA_ARGS__); \
        else if (load == kLoad16Direct) FPNGB_LAUNCH16_ONE(4, kLoad16Direct, FPNGB_TARGS(R, true), kernel, smemfn, grid, threads, __VA_ARGS__); \
        else FPNGB_LAUNCH16_ONE(4, kLoad16Staged, FPNGB_TARGS(R, true), kernel, smemfn, grid, threads, __VA_ARGS__); \
    } while (0)

void launch_scan16(const ScanParams& p, uint32_t n, uint32_t chans, cudaStream_t s)
{
    // one scanline per warp: the multi-scanline sequence that pays off in the pack kernel measured neutral (RGB) to 4 % slower (RGBA) here
    const int load = load16_mode(p, chans);
    dim3 grid((p.h + kScan16Rows - 1) / kScan16Rows, n);
    if (chans == 4 && p.lit1_rule) FPNGB_LAUNCH16_LIT1(row_scan16_kernel, false, scan16_smem, grid, 32 * kScan16Rows, p);
    else FPNGB_LAUNCH16(row_scan16_kernel, false, scan16_smem, grid, 32 * kScan16Rows, p);
}

void launch_hist16(const ScanParams& p, uint32_t n, uint32_t chans, cudaStream_t s)
{
    const int load = load16_mode(p, chans);
    dim3 grid((p.h + kScan16Rows - 1) / kScan16Rows, n);
    FPNGB_LAUNCH16(row_hist16_kernel, false, hist16_smem, grid, 32 * kScan16Rows, p);
}

void launch_pack16(const PackParams& p, uint32_t n, uint32_t chans, cudaStream_t s)
{
    const int load = load16_mode(p, chans);
    const uint32_t rpw = rows_per_warp16(n, p.h), rows_per_cta = pack16_warps(chans) * rpw;
    dim3 grid((p.h + rows_per_cta - 1) / rows_per_cta, n);
    if (chans == 4 && p.lit1_rule) FPNGB_LAUNCH16_LIT1(pack_rows16_kernel, false, pack16_smem, grid, 32 * pack16_warps(chans), p, rpw);
    else FPNGB_LAUNCH16(pack_rows16_kernel, false, pack16_smem, grid, 32 * pack16_warps(chans), p, rpw);
}

// Ragged launches: one per (chans, loader) class, over the class's CTAs (the host sums them per image: ceil(h / rows per CTA)).
uint32_t scan16_rows_per_cta() { return kScan16Rows; }
uint32_t pack16_rows_per_warp(size_t total_rows)
{
    if (g_rows_per_warp_override) return g_rows_per_warp_override;
    return total_rows >= (size_t)sm_count() * 64u * kRowsPerWarp16 ? kRowsPerWarp16 : 1u;
}
uint32_t pack16_rows_per_cta(uint32_t rows_per_warp, uint32_t chans) { return pack16_warps(chans) * rows_per_warp; }

void launch_scan16_ragged(const RaggedParams<ScanParams>& p, uint32_t ctas, uint32_t chans, int load, cudaStream_t s)
{
    if (chans == 4 && p.lit1_rule) FPNGB_LAUNCH16_LIT1(row_scan16_kernel, true, scan16_smem, ctas, 32 * kScan16Rows, p);
    else FPNGB_LAUNCH16(row_scan16_kernel, true, scan16_smem, ctas, 32 * kScan16Rows, p);
}

void launch_hist16_ragged(const RaggedParams<ScanParams>& p, uint32_t ctas, uint32_t chans, int load, cudaStream_t s)
{
    FPNGB_LAUNCH16(row_hist16_kernel, true, hist16_smem, ctas, 32 * kScan16Rows, p);
}

void launch_pack16_ragged(const RaggedParams<PackParams>& p, uint32_t ctas, uint32_t chans, int load, uint32_t rows_per_warp, cudaStream_t s)
{
    if (chans == 4 && p.lit1_rule) FPNGB_LAUNCH16_LIT1(pack_rows16_kernel, true, pack16_smem, ctas, 32 * pack16_warps(chans), p, rows_per_warp);
    else FPNGB_LAUNCH16(pack_rows16_kernel, true, pack16_smem, ctas, 32 * pack16_warps(chans), p, rows_per_warp);
}

}  // namespace fpngb
