// fpng_b200/csrc/png_encode_kernels.cu -- sm_90a kernels of fpngb_encode_png_ragged_device for the images fpng's format does not
// cover: gray8, gray+alpha 8, and 16-bit gray, gray+alpha, RGB and RGBA (B = 1, 2, 2, 4, 6, 8 bytes per pixel).  The file format
// is fixed in include/fpng_b200.h and DESIGN §4.6.
//
//   png_row_kernel<B, ES, kPngHist>  per row: the five filter costs (warp reduction), the chosen filter id, the tokens of the
//                                    filtered row and the image's 288-bin histogram (shared memory, then global)
//   huffman_build_kernel<true, true> per image: fpng's 2-pass code construction with the distance table of B (huffman_kernels.cu)
//   png_row_kernel<B, ES, kPngBits>  per row: the row's code bits under the image's book
//   png_offsets_kernel               per image: exclusive scan of the row bits, compressed-vs-stored decision, container, IEND
//   png_row_kernel<B, ES, kPngPack>  per row: the codes at the row's bit offset (or the raw row of a stored file), row Adler
//   adler_finalize_kernel / idat_crc_stream_kernel (the fpng kernels at each file's header length L: 41 bytes, or more for a label
//                                    map's PLTE and tRNS)
//
// A row is one warp's: lanes take consecutive pixels, 32 per step.  Runs of equal filtered pixels are found with a ballot of the
// pixels that differ from their left neighbour, carried across steps; every token is written by the lane of the pixel it ends on
// (a full match of floor(258 / B) pixels), or by the pixel that ends the run (the run's remainder), so no lane looks ahead.
// The pack kernel re-tokenises the rows instead of reading stored tokens (DESIGN §4.6).
//
// LZ77 mode (FPNGB_LZ77_CHAIN) uses two more modes of the row kernel, also for RGB8 and RGBA8: kPngFilt chooses the filter as
// kPngHist does and writes the filtered row, filter byte first, into the image's stream S with the row's Adler partials;
// kPngRaw writes the raw rows of the images that fell back to stored blocks.  lz77_kernels.cu tokenises and packs S.
#include "row_walk.cuh"
#include "kernels.cuh"

namespace fpngb {

constexpr int kPngRows = 8;                       // warps (scanlines) per CTA
constexpr int kPngStageWords = 136;               // >= (31 + 32 * 116 + 12) / 32 + 1: one step's codes, 116 bits per lane at most
enum { kPngHist = 0, kPngBits = 1, kPngPack = 2, kPngFilt = 3, kPngRaw = 4 };

uint32_t png_rows_per_cta() { return kPngRows; }

__device__ __forceinline__ uint32_t byte_of(uint2 v, int i) { return ((i < 4 ? v.x : v.y) >> (8 * (i & 3))) & 0xFFu; }
__device__ __forceinline__ uint2 shfl_up2(uint2 v) { return make_uint2(__shfl_up_sync(kFullMask, v.x, 1), __shfl_up_sync(kFullMask, v.y, 1)); }
__device__ __forceinline__ uint2 shfl_last2(uint2 v) { return make_uint2(__shfl_sync(kFullMask, v.x, 31), __shfl_sync(kFullMask, v.y, 31)); }

// Pixel x of a scanline in PNG byte order: sample c at row + x * ps + c * cs, ES bytes each, 16-bit samples big-endian.
template <int B, int ES>
__device__ __forceinline__ uint2 load_png_px(const uint8_t* row, uint32_t x, uint32_t ps, unsigned long long cs)
{
    uint32_t wd[2] = {0u, 0u};
#pragma unroll
    for (int c = 0; c < B / ES; c++) {
        const uint8_t* q = row + (size_t)x * ps + (size_t)c * cs;
        if (ES == 1) wd[c >> 2] |= (uint32_t)__ldg(q) << (8 * (c & 3));
        else {
            const uint32_t v = __ldg(reinterpret_cast<const uint16_t*>(q));
            wd[(2 * c) >> 2] |= ((v >> 8) | ((v & 0xFFu) << 8)) << (8 * ((2 * c) & 3));
        }
    }
    return make_uint2(wd[0], wd[1]);
}

__device__ __forceinline__ uint32_t paeth_pred(uint32_t a, uint32_t b, uint32_t c)
{
    const int pa = abs((int)b - (int)c), pb = abs((int)a - (int)c), pc = abs((int)a + (int)b - 2 * (int)c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

__device__ __forceinline__ uint32_t filter_byte(uint32_t type, uint32_t x, uint32_t a, uint32_t b, uint32_t c)
{
    uint32_t pred = 0;
    if (type == 1) pred = a;
    else if (type == 2) pred = b;
    else if (type == 3) pred = (a + b) >> 1;
    else if (type == 4) pred = paeth_pred(a, b, c);
    return (x - pred) & 0xFFu;
}

// x filtered with `type` (a: left, b: up, c: up-left), bytewise at distance B
template <int B>
__device__ __forceinline__ uint2 filter_png_px(uint32_t type, uint2 x, uint2 a, uint2 b, uint2 c)
{
    uint32_t wd[2] = {0u, 0u};
#pragma unroll
    for (int i = 0; i < B; i++) wd[i >> 2] |= filter_byte(type, byte_of(x, i), byte_of(a, i), byte_of(b, i), byte_of(c, i)) << (8 * (i & 3));
    return make_uint2(wd[0], wd[1]);
}

// adds sum min(f, 256 - f) over the filtered bytes f of each of the five filters
template <int B>
__device__ __forceinline__ void add_filter_costs(uint2 x, uint2 a, uint2 b, uint2 c, uint32_t (&cost)[5])
{
#pragma unroll
    for (int i = 0; i < B; i++) {
        const uint32_t xb = byte_of(x, i), ab = byte_of(a, i), bb = byte_of(b, i), cb = byte_of(c, i);
#pragma unroll
        for (uint32_t t = 0; t < 5; t++) { const uint32_t f = filter_byte(t, xb, ab, bb, cb); cost[t] += f < 128u ? f : 256u - f; }
    }
}

// distance code d(B) (a 1-bit code 0) and its extra bit: 1 bit for B = 1, 2, 4; "0" + extra bit 1 for B = 6 (5 + 1), 8 (7 + 1)
template <int B> struct PngDist { static constexpr uint32_t bits = B > 4 ? 2u : 1u, val = B > 4 ? 2u : 0u; };

struct HistSink {
    uint32_t* s_hist;
    __device__ __forceinline__ void lit(uint32_t v) { atomicAdd(&s_hist[v], 1u); }
    __device__ __forceinline__ void match(uint32_t L) { uint32_t s, xb, xv; deflate_len_code(L, s, xb, xv); atomicAdd(&s_hist[s], 1u); }
};

template <int B>
struct BitsSink {
    const uint32_t* s_lit; const uint32_t* s_len; uint32_t bits;
    __device__ __forceinline__ void lit(uint32_t v) { bits += s_lit[v] >> 16; }
    __device__ __forceinline__ void match(uint32_t L)
    {
        uint32_t s, xb, xv; deflate_len_code(L, s, xb, xv);
        bits += (s_len[s - 257] >> 16) + xb + PngDist<B>::bits;
    }
};

// LSB-first bits into a warp's shared staging words (zero outside the live range), OR-ed because lanes share words
template <int B>
struct PutSink {
    const uint32_t* s_lit; const uint32_t* s_len; uint32_t* stage;
    unsigned long long acc; uint32_t nacc, wpos;
    __device__ __forceinline__ void begin(uint32_t bitpos) { acc = 0; nacc = bitpos & 31u; wpos = bitpos >> 5; }
    __device__ __forceinline__ void put(uint32_t code, uint32_t len)
    {
        acc |= (unsigned long long)code << nacc;
        nacc += len;
        if (nacc >= 32u) { atomicOr(&stage[wpos++], (uint32_t)acc); acc >>= 32; nacc -= 32u; }
    }
    __device__ __forceinline__ void end() { if (nacc && (uint32_t)acc) atomicOr(&stage[wpos], (uint32_t)acc); }
    __device__ __forceinline__ void lit(uint32_t v) { const uint32_t e = s_lit[v]; put(e & 0xFFFFu, e >> 16); }
    __device__ __forceinline__ void match(uint32_t L)
    {
        uint32_t s, xb, xv; deflate_len_code(L, s, xb, xv);
        const uint32_t e = s_len[s - 257], sz = e >> 16;
        put((e & 0xFFFFu) | (xv << sz) | (PngDist<B>::val << (sz + xb)), sz + xb + PngDist<B>::bits);
    }
};

// The tokens pixel x emits, in stream order (see the file comment).  eq: x equals its left neighbour (filtered); zb: the last
// pixel before x that does not; fl: x's left neighbour.
template <int B, class Sink>
__device__ __forceinline__ void pixel_tokens(Sink& k, bool eq, uint32_t x, uint32_t w, uint32_t zb, uint2 fx, uint2 fl)
{
    constexpr uint32_t M = 258u / B, minr = (3u + B - 1u) / B;
    auto tail = [&](uint32_t rem, uint2 v) {
        if (rem >= minr) k.match(rem * B);
        else for (uint32_t r = 0; r < rem; r++) {
#pragma unroll
            for (int j = 0; j < B; j++) k.lit(byte_of(v, j));
        }
    };
    if (!eq) {
        if (x > 0) tail((x - 1u - zb) % M, fl);              // the remainder of the run that ends at x - 1 (0: no run)
#pragma unroll
        for (int j = 0; j < B; j++) k.lit(byte_of(fx, j));
    } else {
        const uint32_t run = x - zb;                          // pixels of the run up to and including x
        if (run % M == 0) k.match(M * B);
        if (x == w - 1u) tail(run % M, fx);
    }
}

template <int B, int ES, int MODE, class P = PngEncParams>
__global__ void __launch_bounds__(32 * kPngRows) png_row_kernel(P p)
{
    __shared__ uint32_t s_hist[MODE == kPngHist ? 288 : 1];
    __shared__ uint32_t s_lit[MODE == kPngHist ? 1 : 256];        // code | size << 16
    __shared__ uint32_t s_len[MODE == kPngHist ? 1 : 29];         // length symbols 257..285: code | size << 16
    __shared__ uint32_t s_stage[MODE == kPngPack ? kPngRows : 1][MODE == kPngPack ? kPngStageWords : 1];

    uint32_t local;
    const uint32_t img = ragged_locate(p.ragged, blockIdx.x, local);
    const ImageDesc& d = p.ragged.desc[img];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t y = local * kPngRows + warp, w = d.w, h = d.h;
    const CodeBook* book = d.book;
    const bool stored = (MODE == kPngPack || MODE == kPngRaw) && p.st[img].stored;
    if (MODE == kPngRaw && !stored) return;
    if (MODE == kPngHist) {
        for (uint32_t i = threadIdx.x; i < 288; i += blockDim.x) s_hist[i] = 0u;
    } else if (!stored && MODE != kPngFilt) {
        for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) s_lit[i] = book->lit[i];
        if (threadIdx.x < 29) s_len[threadIdx.x] = book->match[threadIdx.x];
        if (MODE == kPngPack) for (uint32_t i = lane; i < kPngStageWords; i += 32) s_stage[warp][i] = 0u;
    }
    __syncthreads();

    if (y < h) {
        const uint8_t* row = d.pixels + (size_t)y * d.row_pitch;
        const uint8_t* up = row - d.row_pitch;                                  // read only for y > 0
        const uint32_t ps = d.chan_stride ? ES : B;
        const unsigned long long cs = d.chan_stride ? d.chan_stride : ES;
        const size_t r = d.row_base + y;
        uint8_t* file = p.out + d.out_ofs;
        const uint32_t bpl = w * B;

        if (stored) {                                                           // filter 0, fpng's stored-block layout
            auto at = [&](unsigned long long i) -> uint32_t {                   // byte i of the row in PNG order
                const unsigned long long x = i / B, j = i - x * B, c = j / ES;
                return __ldg(row + x * ps + c * cs + (ES == 2 ? 1u - (uint32_t)(j & 1u) : 0u));
            };
            store_row_raw(at, file + d.hdr_len, y, bpl, lane, &p.row_adler[r]);
            return;
        }

        uint32_t ft;
        if (MODE == kPngHist || MODE == kPngFilt) {                                                 // the filter with the smallest cost, ties to the lower id
            uint32_t cost[5] = {0u, 0u, 0u, 0u, 0u};
            uint2 ca = make_uint2(0u, 0u), cc = ca;
            for (uint32_t x0 = 0; x0 < w; x0 += 32) {
                const uint32_t x = x0 + lane;
                const bool valid = x < w;
                const uint2 cx = valid ? load_png_px<B, ES>(row, x, ps, cs) : make_uint2(0u, 0u);
                const uint2 bx = (valid && y) ? load_png_px<B, ES>(up, x, ps, cs) : make_uint2(0u, 0u);
                uint2 a = shfl_up2(cx), c = shfl_up2(bx);
                if (lane == 0) { a = ca; c = cc; }
                ca = shfl_last2(cx); cc = shfl_last2(bx);
                if (valid) add_filter_costs<B>(cx, a, bx, c, cost);
            }
            unsigned long long best = warp_sum_u64(cost[0]);
            ft = 0;
#pragma unroll
            for (uint32_t t = 1; t < 5; t++) { const unsigned long long v = warp_sum_u64(cost[t]); if (v < best) { best = v; ft = t; } }
            if (lane == 0) p.row_filter[r] = (uint8_t)ft;
        } else {
            ft = p.row_filter[r];
        }

        if constexpr (MODE == kPngFilt) {                                       // S row: filter byte, filtered bytes; Adler partials
            uint8_t* srow = p.lz_s + d.lz_ofs + (unsigned long long)y * (bpl + 1u);
            unsigned long long s1 = 0, si = 0;
            uint2 ca = make_uint2(0u, 0u), cc = ca;
            for (uint32_t x0 = 0; x0 < w; x0 += 32) {
                const uint32_t x = x0 + lane;
                const bool valid = x < w;
                const uint2 cx = valid ? load_png_px<B, ES>(row, x, ps, cs) : make_uint2(0u, 0u);
                const uint2 bx = (valid && y) ? load_png_px<B, ES>(up, x, ps, cs) : make_uint2(0u, 0u);
                uint2 a = shfl_up2(cx), c = shfl_up2(bx);
                if (lane == 0) { a = ca; c = cc; }
                ca = shfl_last2(cx); cc = shfl_last2(bx);
                if (valid) {
                    const uint2 fx = filter_png_px<B>(ft, cx, a, bx, c);
#pragma unroll
                    for (int j = 0; j < B; j++) {
                        const uint32_t v = byte_of(fx, j);
                        srow[1u + x * B + j] = (uint8_t)v;
                        s1 += v; si += (1ull + (unsigned long long)x * B + j) * v;
                    }
                }
            }
            s1 = warp_sum_u64(s1); si = warp_sum_u64(si);
            if (lane == 0) {
                srow[0] = (uint8_t)ft;
                const unsigned long long S1 = s1 + ft, n = (unsigned long long)bpl + 1ull;
                p.row_adler[r] = make_uint2((uint32_t)(S1 % kAdlerMod), (uint32_t)((n * S1 - si) % kAdlerMod));
            }
            return;
        }

        HistSink hs{s_hist};
        BitsSink<B> bsink{s_lit, s_len, 0u};
        PutSink<B> put{s_lit, s_len, s_stage[MODE == kPngPack ? warp : 0]};
        unsigned long long s1 = 0, si = 0;                                      // Adler partials: sum v, sum (1 + byte index) v
        const unsigned long long G = MODE == kPngPack ? p.row_ofs[r] : 0ull;
        uint32_t* file_words = reinterpret_cast<uint32_t*>(file);
        const unsigned long long first_word = G >> 5;
        unsigned long long gword = first_word;
        uint32_t fill = (uint32_t)(G & 31ull);

        uint2 ca = make_uint2(0u, 0u), cc = ca, cf = ca;
        uint32_t cz = 0;                                                        // last pixel of earlier steps that differs from its left
        for (uint32_t x0 = 0; x0 < w; x0 += 32) {
            const uint32_t x = x0 + lane;
            const bool valid = x < w;
            const uint2 cx = valid ? load_png_px<B, ES>(row, x, ps, cs) : make_uint2(0u, 0u);
            const uint2 bx = (valid && y) ? load_png_px<B, ES>(up, x, ps, cs) : make_uint2(0u, 0u);
            uint2 a = shfl_up2(cx), c = shfl_up2(bx);
            if (lane == 0) { a = ca; c = cc; }
            const uint2 fx = valid ? filter_png_px<B>(ft, cx, a, bx, c) : make_uint2(0u, 0u);
            uint2 fl = shfl_up2(fx);
            if (lane == 0) fl = cf;
            const bool eq = valid && x > 0 && fx.x == fl.x && fx.y == fl.y;
            const uint32_t nm = __ballot_sync(kFullMask, valid && !eq);
            const uint32_t below = nm & ((1u << lane) - 1u);
            const uint32_t zb = below ? x0 + 31u - __clz(below) : cz;
            if (nm) cz = x0 + 31u - __clz(nm);
            ca = shfl_last2(cx); cc = shfl_last2(bx); cf = shfl_last2(fx);

            if (MODE == kPngHist) {
                if (x0 == 0 && lane == 0) hs.lit(ft);
                if (valid) pixel_tokens<B>(hs, eq, x, w, zb, fx, fl);
            } else {
                const uint32_t fbits = (x0 == 0 && lane == 0) ? s_lit[ft] >> 16 : 0u;
                bsink.bits = MODE == kPngBits ? bsink.bits + fbits : fbits;     // bits: the lane's whole row; pack: this step
                if (valid) pixel_tokens<B>(bsink, eq, x, w, zb, fx, fl);
                if (MODE == kPngPack) {
#pragma unroll
                    for (int j = 0; j < B; j++) { const uint32_t v = byte_of(fx, j); s1 += v; si += (1ull + (unsigned long long)x * B + j) * v; }
                    uint32_t step_bits;
                    const uint32_t ofs = warp_excl_scan_u32(bsink.bits, lane, step_bits);
                    put.begin(fill + ofs);
                    if (x0 == 0 && lane == 0) put.lit(ft);
                    if (valid) pixel_tokens<B>(put, eq, x, w, zb, fx, fl);
                    put.end();
                    __syncwarp();
                    // flush whole words; the row's first word is shared with the previous row or the block header
                    uint32_t* stage = put.stage;
                    fill += step_bits;
                    const uint32_t nwords = fill >> 5;
                    const uint32_t leftover = stage[nwords];
                    for (uint32_t j = lane; j < nwords; j += 32) {
                        const uint32_t v = stage[j];
                        if (gword + j == first_word) atomicOr(&file_words[gword + j], v);
                        else file_words[gword + j] = v;
                    }
                    __syncwarp();
                    for (uint32_t j = lane; j <= nwords; j += 32) stage[j] = j == 0 ? leftover : 0u;
                    __syncwarp();
                    gword += nwords;
                    fill &= 31u;
                }
            }
        }
        if (MODE == kPngBits) {
            const uint32_t rb = warp_sum_u32(bsink.bits);
            if (lane == 0) p.row_bits[r] = rb;
        }
        if (MODE == kPngPack) {
            if (lane == 0 && fill) { const uint32_t v = put.stage[0]; if (v) atomicOr(&file_words[gword], v); }
            s1 = warp_sum_u64(s1); si = warp_sum_u64(si);
            if (lane == 0) {
                const unsigned long long S1 = s1 + ft, n = (unsigned long long)bpl + 1ull;
                p.row_adler[r] = make_uint2((uint32_t)(S1 % kAdlerMod), (uint32_t)((n * S1 - si) % kAdlerMod));
            }
        }
    }

    if (MODE == kPngHist) {
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < 288; i += blockDim.x)
            if (s_hist[i]) atomicAdd(&p.hist[(size_t)img * 288 + i], s_hist[i]);
    }
}

__device__ __forceinline__ void store_be32_png(uint8_t* q, uint32_t v)
{
    q[0] = (uint8_t)(v >> 24); q[1] = (uint8_t)(v >> 16); q[2] = (uint8_t)(v >> 8); q[3] = (uint8_t)v;
}

// Image blockIdx.x of p.desc: row bit offsets, the compressed-vs-stored decision (stored iff FPNGB_FORCE_UNCOMPRESSED or the
// compressed zlib stream would be longer), the L-byte container header (L = hdr_len) with the IDAT length at L - 8, the zlib and
// block headers, the stored block headers or the end-of-block code, the IEND chunk and the file size (0 for a label map with an
// out-of-range id: the file is written in its slot all the same, and read by nothing).  Zeroes the words neighbouring rows share.
// LZ (P = PngLzParams): the units are the image's segments of S (seg_bits / seg_ofs) instead of its rows.
template <class P>
__device__ __forceinline__ void png_offsets_body(const P& p)
{
    constexpr bool LZ = std::is_same<P, PngLzParams>::value;
    __shared__ unsigned long long s_warp[kOffsetsThreads / 32];
    const uint32_t img = blockIdx.x, tid = threadIdx.x;
    const ImageDesc& d = p.desc[img];
    const CodeBook* book = d.book;
    const uint32_t h = d.h, hdr_bits = book->hdr_bits, L = d.hdr_len;
    const unsigned long long base = 8ull * L + hdr_bits;
    const uint32_t* row_bits;
    unsigned long long* row_ofs;
    uint32_t units;
    if constexpr (LZ) { row_bits = p.seg_bits + d.seg_base; row_ofs = p.seg_ofs + d.seg_base; units = d.nseg; }
    else { row_bits = p.row_bits + d.row_base; row_ofs = p.row_ofs + d.row_base; units = h; }
    uint8_t* file = p.out + d.out_ofs;
    uint32_t* file_words = reinterpret_cast<uint32_t*>(file);
    ImageState* st = p.st + img;

    unsigned long long running = 0;
    for (uint32_t y0 = 0; y0 < units; y0 += blockDim.x) {
        const uint32_t y = y0 + tid;
        unsigned long long tot;
        const unsigned long long ex = block_excl_scan_u64(y < units ? row_bits[y] : 0ull, s_warp, tot);
        if (y < units) row_ofs[y] = base + running + ex;
        running += tot;
    }
    const unsigned long long raw = ((unsigned long long)d.w * d.chans + 1ull) * h, nblk = (raw + 65534ull) / 65535ull;
    const unsigned long long zstored = 2ull + raw + 5ull * nblk + 4ull;
    const unsigned long long zcomp = (hdr_bits + running + (book->eob >> 16) + 7ull) / 8ull + 4ull;
    const bool compressed = !(p.flags & 2u) && zcomp <= zstored;
    const uint32_t zsize = (uint32_t)(compressed ? zcomp : zstored);

    __syncthreads();
    if (compressed) {
        for (uint32_t y = 1 + tid; y < units; y += blockDim.x) file_words[row_ofs[y] >> 5] = 0u;
        const unsigned long long e = base + running;
        if (tid == 0) { file_words[e >> 5] = 0u; file_words[(e >> 5) + 1] = 0u; }
    }
    __syncthreads();
    const uint32_t hbytes = compressed ? (hdr_bits + 7u) >> 3 : 2u;
    const uint32_t hend = compressed ? 4u * ((uint32_t)(base >> 5) + 1u) : L + 2u;
    const uint8_t* hdr = p.headers + d.hdr_at;
    for (uint32_t i = tid; i < hend; i += blockDim.x) {
        uint8_t v = 0;
        if (i < L) v = hdr[i];
        else if (i - L < hbytes) v = compressed ? book->hdr[i - L] : (i == L ? 0x78 : 0x01);
        if (i >= L - 8u && i < L - 4u) v = (uint8_t)(zsize >> (8 * (L - 5u - i)));
        file[i] = v;
    }
    if (!compressed) {
        for (unsigned long long j = tid; j < nblk; j += blockDim.x) {
            uint8_t* b = file + L + 2ull + j * 65540ull;
            const unsigned long long remaining = raw - j * 65535ull;
            const uint32_t len = remaining < 65535ull ? (uint32_t)remaining : 65535u;
            b[0] = (j + 1 == nblk) ? 1 : 0;
            b[1] = (uint8_t)len; b[2] = (uint8_t)(len >> 8);
            b[3] = (uint8_t)~len; b[4] = (uint8_t)(~len >> 8);
        }
    }
    __syncthreads();
    if (tid == 0) {
        if (compressed) {
            const unsigned long long e = base + running;
            const unsigned long long v = (unsigned long long)(book->eob & 0xFFFFu) << (e & 7ull);
            uint8_t* q = file + (e >> 3);
            for (int i = 0; i < 3; i++) { const uint8_t b = (uint8_t)(v >> (8 * i)); if (b) q[i] |= b; }
        }
        static const uint8_t iend[12] = { 0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82 };
        uint8_t* t = file + L + zsize;
        store_be32_png(t, 0u);
        for (int i = 0; i < 12; i++) t[4 + i] = iend[i];
        st->zsize = zsize;
        st->stored = compressed ? 0u : 1u;
        st->crc_acc = 0u;
        st->tiles_done = 0u;
        st->status = 0u;
        p.sizes[d.index] = (p.bad && p.bad[d.index]) ? 0u : L + zsize + kPngTrailerSize;
    }
}

__global__ void __launch_bounds__(kOffsetsThreads) png_offsets_kernel(PngEncParams p) { png_offsets_body(p); }
__global__ void __launch_bounds__(kOffsetsThreads) png_lz_offsets_kernel(PngLzParams p) { png_offsets_body(p); }

template <int B, int ES>
static void launch_rows_t(const PngEncParams& p, uint32_t ctas, int mode, cudaStream_t s)
{
    if (mode == kPngHist) png_row_kernel<B, ES, kPngHist><<<ctas, 32 * kPngRows, 0, s>>>(p);
    else if (mode == kPngBits) png_row_kernel<B, ES, kPngBits><<<ctas, 32 * kPngRows, 0, s>>>(p);
    else png_row_kernel<B, ES, kPngPack><<<ctas, 32 * kPngRows, 0, s>>>(p);
}

void launch_png_rows(const PngEncParams& p, uint32_t ctas, uint32_t bpp, uint32_t depth, int mode, cudaStream_t s)
{
    switch (bpp) {
    case 1: launch_rows_t<1, 1>(p, ctas, mode, s); break;
    case 2: if (depth == 8) launch_rows_t<2, 1>(p, ctas, mode, s); else launch_rows_t<2, 2>(p, ctas, mode, s); break;
    case 4: launch_rows_t<4, 2>(p, ctas, mode, s); break;
    case 6: launch_rows_t<6, 2>(p, ctas, mode, s); break;
    default: launch_rows_t<8, 2>(p, ctas, mode, s); break;
    }
}

void launch_png_offsets(const PngEncParams& p, uint32_t n, cudaStream_t s)
{
    png_offsets_kernel<<<n, kOffsetsThreads, 0, s>>>(p);
}

template <int B, int ES>
static void launch_lz_rows_t(const PngLzParams& p, uint32_t ctas, int mode, cudaStream_t s)
{
    if (mode == 0) png_row_kernel<B, ES, kPngFilt, PngLzParams><<<ctas, 32 * kPngRows, 0, s>>>(p);
    else png_row_kernel<B, ES, kPngRaw><<<ctas, 32 * kPngRows, 0, s>>>(p);
}

void launch_png_lz_rows(const PngLzParams& p, uint32_t ctas, uint32_t bpp, uint32_t depth, int mode, cudaStream_t s)
{
    switch (bpp) {
    case 1: launch_lz_rows_t<1, 1>(p, ctas, mode, s); break;
    case 2: if (depth == 8) launch_lz_rows_t<2, 1>(p, ctas, mode, s); else launch_lz_rows_t<2, 2>(p, ctas, mode, s); break;
    case 3: launch_lz_rows_t<3, 1>(p, ctas, mode, s); break;
    case 4: if (depth == 8) launch_lz_rows_t<4, 1>(p, ctas, mode, s); else launch_lz_rows_t<4, 2>(p, ctas, mode, s); break;
    case 6: launch_lz_rows_t<6, 2>(p, ctas, mode, s); break;
    default: launch_lz_rows_t<8, 2>(p, ctas, mode, s); break;
    }
}

void launch_png_lz_offsets(const PngLzParams& p, uint32_t n, cudaStream_t s)
{
    png_lz_offsets_kernel<<<n, kOffsetsThreads, 0, s>>>(p);
}

}  // namespace fpngb
