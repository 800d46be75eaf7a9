// fpng_b200/csrc/encode_kernels.cu -- sm_90a kernels of the fpng encode hot path.
//
//   K1  row_scan_kernel     filter + RLE match scan + per-row bit count + per-row Adler-32 partials
//                           (or, for 2-pass mode, the 288-bin literal/length histogram)
//   K2  row_offsets_kernel  exclusive scan of row bit counts -> row bit offsets; compressed-vs-stored decision
//                           (fpng.cpp:567-588,1705,1728); writes the 58-byte container header, the block header,
//                           EOB, IEND and zeroes the words shared between neighbouring rows
//   K3  pack_rows_kernel    re-tokenises each row and writes its Huffman codes at the row's bit offset
//                           (stored-block fallback: strided copy with 5-byte block headers, fpng.cpp:818-866)
//   K3b adler_finalize_kernel  combines the per-row (S1,S2) partials into the zlib Adler-32 (big-endian)
//
// All are HBM/L2-bound byte kernels: no tensor cores (there is no contraction anywhere in this path).
#include "row_walk.cuh"
#include "kernels.cuh"

namespace fpngb {

// ------------------------------------------------------------------------------------------------
// K1: scan
// ------------------------------------------------------------------------------------------------
template <int CHANS>
__device__ __forceinline__ uint32_t literal_bits(const uint8_t* s_lit, uint32_t px)
{
    uint32_t b = s_lit[px & 0xFF] + s_lit[(px >> 8) & 0xFF] + s_lit[(px >> 16) & 0xFF];
    if (CHANS == 4) b += s_lit[px >> 24];
    return b;
}

template <int CHANS, int MODE, bool HIST>
__global__ void __launch_bounds__(kScanThreads) row_scan_kernel(ScanParams p)
{
    __shared__ uint8_t s_lit[256];
    __shared__ uint8_t s_match[88];
    __shared__ uint32_t s_hist[HIST ? 288 : 1];

    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t img = blockIdx.y;
    const uint32_t y = blockIdx.x * kRowsPerBlock + warp;
    const CodeBook* book = p.books + (size_t)img * p.book_stride;

    if (HIST) {
        for (uint32_t i = threadIdx.x; i < 288; i += blockDim.x) s_hist[i] = 0;
    } else {
        for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) s_lit[i] = book->lit_size[i];
        if (threadIdx.x < 88) s_match[threadIdx.x] = book->match_bits[threadIdx.x];
    }
    __syncthreads();

    if (y < p.h) {
        const uint32_t w = p.w, bpl = w * CHANS;
        const uint8_t* cur = p.pixels + (size_t)img * p.image_stride + (size_t)y * bpl;
        const uint8_t* prev = y ? cur - bpl : nullptr;
        const uint32_t filt = y ? 2u : 0u;
        const uint32_t nsteps = (w + kPixPerStep - 1) / kPixPerStep;

        RowCarry carry = { 0u, 0u };
        uint32_t bits = 0, sumA = 0;
        unsigned long long sumB = 0;

        for (uint32_t step = 0; step < nsteps; step++) {
            const uint32_t p0 = step * kPixPerStep + lane * kPixPerLane;
            const uint32_t bo = p0 * CHANS;
            LaneTokens t;
            uint32_t dw[CHANS];
            t.nvp = p0 < w ? min(4u, w - p0) : 0u;
            load_filtered_step<CHANS, MODE>(cur, prev, bo, bpl, dw, t.px);
            classify_step<CHANS>(t, p0, w, carry, lane);

            if (HIST) {
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    if (t.mlen[k]) { uint32_t s, xb, xv; deflate_len_code(t.mlen[k] * CHANS, s, xb, xv); atomicAdd(&s_hist[s], 1u); }
                    if (t.litmask & (1u << k)) {
                        atomicAdd(&s_hist[t.px[k] & 0xFF], 1u);
                        atomicAdd(&s_hist[(t.px[k] >> 8) & 0xFF], 1u);
                        atomicAdd(&s_hist[(t.px[k] >> 16) & 0xFF], 1u);
                        if (CHANS == 4) atomicAdd(&s_hist[t.px[k] >> 24], 1u);
                    }
                }
                if (t.tail) { uint32_t s, xb, xv; deflate_len_code(t.tail * CHANS, s, xb, xv); atomicAdd(&s_hist[s], 1u); }
            } else {
                // RGBA 1-pass "one-pixel match vs four literals" (fpng.cpp:1520-1528): a match token of exactly one pixel costs
                // min(match, literals) -- strictly: literals are taken iff match bits > literal bits.  Only compiled into the
                // rule-aware instantiation; p.lit1_rule is warp-uniform.
                uint32_t tail_cost = s_match[t.tail];
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    uint32_t mc = s_match[t.mlen[k]];
                    if (CHANS == 4 && p.lit1_rule && t.mlen[k] == 1u) { const uint32_t lb = literal_bits<CHANS>(s_lit, run_pixel_before(t, k)); if (mc > lb) mc = lb; }
                    bits += mc;
                    if (t.litmask & (1u << k)) bits += literal_bits<CHANS>(s_lit, t.px[k]);
                }
                if (CHANS == 4 && p.lit1_rule && t.tail == 1u) { const uint32_t lb = literal_bits<CHANS>(s_lit, run_pixel_before(t, t.nvp)); if (tail_cost > lb) tail_cost = lb; }
                bits += tail_cost;

                // Adler-32 partials over the filtered bytes (fpng.cpp:403-487 computes the same sum serially)
                uint32_t t1 = 0, t2 = 0;
#pragma unroll
                for (int i = 0; i < CHANS; i++) {
                    t1 = __dp4a(dw[i], 0x01010101u, t1);
                    t2 = __dp4a(dw[i], 0x03020100u + 0x04040404u * i, t2);
                }
                sumA += t1;
                sumB += (unsigned long long)bo * t1 + t2;

                // capacity rule needs the size of the row's last flush unit (SURVEY Q5)
                if (t.nvp > 0 && p0 + t.nvp == w && y == p.h - 1) {
                    const uint32_t k = t.nvp - 1;
                    uint32_t lu;
                    if (t.tail) lu = tail_cost;
                    else if (!(t.litmask & (1u << k))) lu = s_match[t.mlen[k]];
                    else lu = literal_bits<CHANS>(s_lit, t.px[k]) + ((w == 1 && p.merge_first_unit) ? s_lit[filt] : 0u);
                    p.st[img].last_unit_bits = lu;
                }
            }
        }

        if (HIST) {
            if (lane == 0) atomicAdd(&s_hist[filt], 1u);
        } else {
            const uint32_t row_bits = warp_sum_u32(bits) + s_lit[filt];
            const unsigned long long A = warp_sum_u64(sumA);
            const unsigned long long B = warp_sum_u64(sumB);
            if (lane == 0) {
                const unsigned long long n = (unsigned long long)bpl + 1ull;
                const unsigned long long S1 = A + filt;
                const unsigned long long S2 = n * S1 - (A + B);   // sum (n - i) x_i, i = 1 + byte offset; filter byte at i = 0
                p.row_bits[(size_t)img * p.h + y] = row_bits;
                p.row_adler[(size_t)img * p.h + y] = make_uint2((uint32_t)(S1 % kAdlerMod), (uint32_t)(S2 % kAdlerMod));
            }
        }
    }

    if (HIST) {
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < 288; i += blockDim.x)
            if (s_hist[i]) atomicAdd(&p.hist[(size_t)img * 288 + i], s_hist[i]);
    }
}

// ------------------------------------------------------------------------------------------------
// K2: offsets + container
// ------------------------------------------------------------------------------------------------

__device__ __forceinline__ void store_be32(uint8_t* p, uint32_t v)
{
    p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v;
}

// RAGGED: image blockIdx.x of p.desc; its descriptor replaces the call-wide shape, book and header, and the row tables, image
// state, size and output are rebased to it (the body then runs as for image 0)
template <bool RAGGED = false>
__global__ void __launch_bounds__(kOffsetsThreads) row_offsets_kernel(OffsetsParams p)
{
    __shared__ unsigned long long s_warp[kOffsetsThreads / 32];
    uint32_t img = blockIdx.x;
    const uint32_t tid = threadIdx.x;
    const uint8_t* ragged_header = nullptr;
    if constexpr (RAGGED) {
        const ImageDesc& d = p.desc[img];
        p.row_bits += d.row_base; p.row_ofs += d.row_base; p.books = d.book; p.book_stride = 0; p.st += img;
        p.out += d.out_ofs; p.sizes += d.index; p.w = d.w; p.h = d.h; p.chans = d.chans;
        ragged_header = d.png_header;
        img = 0;
    }
    const CodeBook* book = p.books + (size_t)img * p.book_stride;
    const uint32_t h = p.h;
    const uint32_t hdr_bits = book->hdr_bits;
    const unsigned long long base = (unsigned long long)kZlibBitBase + hdr_bits;
    uint8_t* file = p.out + (size_t)img * p.out_stride;
    uint32_t* file_words = reinterpret_cast<uint32_t*>(file);
    ImageState* st = p.st + img;

    // exclusive scan of row bit counts
    unsigned long long running = 0;
    for (uint32_t y0 = 0; y0 < h; y0 += blockDim.x) {
        const uint32_t y = y0 + tid;
        const unsigned long long v = y < h ? p.row_bits[(size_t)img * h + y] : 0ull;
        unsigned long long tot;
        const unsigned long long ex = block_excl_scan_u64(v, s_warp, tot);
        if (y < h) p.row_ofs[(size_t)img * h + y] = base + running + ex;
        running += tot;
    }
    const unsigned long long row_bits_total = running;

    // compressed-vs-stored decision: the reference gives up iff a PUT_BITS_FLUSH would see dst_ofs + 8 > cap
    // (fpng.cpp:567-576; dst_ofs is monotone so only the last flush matters) or the final bytes + Adler do not fit.
    const unsigned long long raw = ((unsigned long long)p.w * p.chans + 1ull) * h;
    const unsigned long long cap = ((kPngHeaderSize + raw + 7ull) & ~7ull) - kPngHeaderSize;      // fpng.cpp:1705
    const uint32_t eob_size = book->eob >> 16;
    const unsigned long long total_bits = hdr_bits + row_bits_total + eob_size;
    const unsigned long long d_last = (hdr_bits + row_bits_total - st->last_unit_bits) >> 3;
    const unsigned long long zbytes = (total_bits + 7ull) >> 3;
    const bool compressed = !(p.flags & 2u) && (d_last + 8ull <= cap) && (zbytes + 4ull <= cap);
    const unsigned long long nblk = (raw + 65534ull) / 65535ull;
    const uint32_t zsize = compressed ? (uint32_t)(zbytes + 4ull) : (uint32_t)(2ull + raw + 5ull * nblk + 4ull);

    __syncthreads();
    if (compressed) {
        // zero every word that two rows (or the last row and the EOB) share; K3 ORs into them
        for (uint32_t y = 1 + tid; y < h; y += blockDim.x) file_words[p.row_ofs[(size_t)img * h + y] >> 5] = 0u;
        const unsigned long long e = base + row_bits_total;
        if (tid == 0) { file_words[e >> 5] = 0u; file_words[(e >> 5) + 1] = 0u; }
    }
    __syncthreads();

    // container header (fpng.cpp:1766-1791) + pre-serialised block header
    // In compressed mode the loop runs to the end of the word that holds row 0's first bit, so that word is
    // initialised (header tail bits, zero elsewhere) before K3 ORs row 0 into it.
    const uint32_t hbytes = compressed ? (hdr_bits + 7u) >> 3 : 2u;
    const uint32_t hend = compressed ? 4u * ((uint32_t)(base >> 5) + 1u) : kPngHeaderSize + 2u;
    for (uint32_t i = tid; i < hend; i += blockDim.x) {
        uint8_t v = 0;
        if (i < kPngHeaderSize) v = RAGGED ? ragged_header[i] : p.png_header[i];
        else if (i - kPngHeaderSize < hbytes) v = compressed ? book->hdr[i - kPngHeaderSize] : (i == kPngHeaderSize ? 0x78 : 0x01);
        if (i >= 50 && i < 54) v = (uint8_t)(zsize >> (8 * (53 - i)));
        file[i] = v;
    }
    if (!compressed) {
        // stored block headers: BFINAL, LEN, ~LEN (fpng.cpp:829-850)
        for (unsigned long long j = tid; j < nblk; j += blockDim.x) {
            uint8_t* b = file + kPngHeaderSize + 2ull + j * 65540ull;
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
            // end-of-block code right after the last row; pad bits stay zero (fpng.cpp:1249-1251)
            const unsigned long long e = base + row_bits_total;
            const unsigned long long v = (unsigned long long)(book->eob & 0xFFFFu) << (e & 7ull);
            uint8_t* q = file + (e >> 3);
            for (int i = 0; i < 3; i++) { const uint8_t b = (uint8_t)(v >> (8 * i)); if (b) q[i] |= b; }
        }
        static const uint8_t iend[12] = { 0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82 };
        uint8_t* t = file + kPngHeaderSize + zsize;
        for (int i = 0; i < 4; i++) t[i] = 0;
        for (int i = 0; i < 12; i++) t[4 + i] = iend[i];
        st->zsize = zsize;
        st->stored = compressed ? 0u : 1u;
        st->crc_acc = 0u;
        st->tiles_done = 0u;
        st->status = 0u;
        p.sizes[img] = kPngHeaderSize + zsize + kPngTrailerSize;
    }
}

// ------------------------------------------------------------------------------------------------
// K3: pack
// ------------------------------------------------------------------------------------------------
struct BitStager {
    uint32_t* stage;            // per-warp shared staging words (zero outside the live range)
    unsigned long long acc;
    uint32_t nacc;              // bits pending in acc (incl. the sub-word offset), < 32 between puts
    uint32_t wpos;
    __device__ __forceinline__ void begin(uint32_t bitpos) { acc = 0; nacc = bitpos & 31u; wpos = bitpos >> 5; }
    __device__ __forceinline__ void put(uint32_t code, uint32_t len)
    {
        acc |= (unsigned long long)code << nacc;
        nacc += len;
        if (nacc >= 32u) { atomicOr(&stage[wpos++], (uint32_t)acc); acc >>= 32; nacc -= 32u; }
    }
    __device__ __forceinline__ void end() { if (nacc && (uint32_t)acc) atomicOr(&stage[wpos], (uint32_t)acc); }
};

template <int CHANS>
__device__ __forceinline__ void put_literal(BitStager& bs, const uint32_t* s_lit, uint32_t px)
{
    const uint32_t c0 = s_lit[px & 0xFF], c1 = s_lit[(px >> 8) & 0xFF], c2 = s_lit[(px >> 16) & 0xFF];
    const uint32_t l0 = c0 >> 16, l1 = c1 >> 16, l2 = c2 >> 16;
    bs.put((c0 & 0xFFFFu) | ((c1 & 0xFFFFu) << l0), l0 + l1);
    if (CHANS == 4) {
        const uint32_t c3 = s_lit[px >> 24], l3 = c3 >> 16;
        bs.put((c2 & 0xFFFFu) | ((c3 & 0xFFFFu) << l2), l2 + l3);
    } else {
        bs.put(c2 & 0xFFFFu, l2);
    }
}

template <int CHANS>
__device__ __forceinline__ uint32_t literal_bits_w(const uint32_t* s_lit, uint32_t px)
{
    uint32_t b = (s_lit[px & 0xFF] >> 16) + (s_lit[(px >> 8) & 0xFF] >> 16) + (s_lit[(px >> 16) & 0xFF] >> 16);
    if (CHANS == 4) b += s_lit[px >> 24] >> 16;
    return b;
}

template <int CHANS, int MODE>
__global__ void __launch_bounds__(kPackThreads) pack_rows_kernel(PackParams p)
{
    __shared__ uint32_t s_lit[256];
    __shared__ uint32_t s_match[88];
    __shared__ uint32_t s_stage[kRowsPerBlock][kStageWords];

    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t img = blockIdx.y;
    const uint32_t y = blockIdx.x * kRowsPerBlock + warp;
    const CodeBook* book = p.books + (size_t)img * p.book_stride;
    const ImageState st = p.st[img];

    if (!st.stored) {
        for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) s_lit[i] = book->lit[i];
        if (threadIdx.x < 88) s_match[threadIdx.x] = book->match[threadIdx.x];
        for (uint32_t i = lane; i < kStageWords; i += 32) s_stage[warp][i] = 0u;
    }
    __syncthreads();
    if (y >= p.h) return;

    const uint32_t w = p.w, bpl = w * CHANS;
    const uint8_t* cur = p.pixels + (size_t)img * p.image_stride + (size_t)y * bpl;
    uint8_t* file = p.out + (size_t)img * p.out_stride;

    if (st.stored) {
        store_row_raw(cur, file + kPngHeaderSize, y, bpl, lane, &p.row_adler[(size_t)img * p.h + y]);
        return;
    }

    const uint8_t* prev = y ? cur - bpl : nullptr;
    uint32_t* file_words = reinterpret_cast<uint32_t*>(file);
    uint32_t* stage = s_stage[warp];
    const unsigned long long G = p.row_ofs[(size_t)img * p.h + y];
    const unsigned long long first_word = G >> 5;
    unsigned long long gword = first_word;      // global word index that stage[0] maps to
    uint32_t fill = (uint32_t)(G & 31ull);       // live bits in the staging buffer
    const uint32_t nsteps = (w + kPixPerStep - 1) / kPixPerStep;
    const uint32_t fcode = s_lit[y ? 2 : 0];

    RowCarry carry = { 0u, 0u };
    for (uint32_t step = 0; step < nsteps; step++) {
        const uint32_t p0 = step * kPixPerStep + lane * kPixPerLane;
        LaneTokens t;
        uint32_t dw[CHANS];
        t.nvp = p0 < w ? min(4u, w - p0) : 0u;
        load_filtered_step<CHANS, MODE>(cur, prev, p0 * CHANS, bpl, dw, t.px);
        classify_step<CHANS>(t, p0, w, carry, lane);

        uint32_t nb = (step == 0 && lane == 0) ? (fcode >> 16) : 0u;
        // bit j < 4: the one-pixel match flushed at slot j is written as four literals; bit 4: same for the row-end token
        // (RGBA 1-pass rule, fpng.cpp:1520-1528; p.lit1_rule is warp-uniform and zero for every other mode)
        uint32_t as_lits = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            uint32_t mc = s_match[t.mlen[k]] >> 24;
            if (CHANS == 4 && p.lit1_rule && t.mlen[k] == 1u) { const uint32_t lb = literal_bits_w<CHANS>(s_lit, run_pixel_before(t, k)); if (mc > lb) { mc = lb; as_lits |= 1u << k; } }
            nb += mc;
            if (t.litmask & (1u << k)) nb += literal_bits_w<CHANS>(s_lit, t.px[k]);
        }
        {
            uint32_t mc = s_match[t.tail] >> 24;
            if (CHANS == 4 && p.lit1_rule && t.tail == 1u) { const uint32_t lb = literal_bits_w<CHANS>(s_lit, run_pixel_before(t, t.nvp)); if (mc > lb) { mc = lb; as_lits |= 16u; } }
            nb += mc;
        }

        uint32_t step_bits;
        const uint32_t ofs = warp_excl_scan_u32(nb, lane, step_bits);

        BitStager bs; bs.stage = stage;
        bs.begin(fill + ofs);
        if (step == 0 && lane == 0) bs.put(fcode & 0xFFFFu, fcode >> 16);
#pragma unroll
        for (int k = 0; k < 4; k++) {
            if (as_lits & (1u << k)) put_literal<CHANS>(bs, s_lit, run_pixel_before(t, k));
            else if (t.mlen[k]) { const uint32_t m = s_match[t.mlen[k]]; bs.put(m & 0xFFFFFFu, m >> 24); }
            if (t.litmask & (1u << k)) put_literal<CHANS>(bs, s_lit, t.px[k]);
        }
        if (as_lits & 16u) put_literal<CHANS>(bs, s_lit, run_pixel_before(t, t.nvp));
        else if (t.tail) { const uint32_t m = s_match[t.tail]; bs.put(m & 0xFFFFFFu, m >> 24); }
        bs.end();
        __syncwarp();

        // flush whole words; the row's first word is shared with the previous row / the block header
        fill += step_bits;
        const uint32_t nwords = fill >> 5;
        const uint32_t leftover = stage[nwords];
        for (uint32_t j = lane; j < nwords; j += 32) {
            const uint32_t v = stage[j];
            if (gword + j == first_word) atomicOr(&file_words[gword + j], v);
            else file_words[gword + j] = v;
        }
        __syncwarp();
        for (uint32_t j = lane; j <= nwords; j += 32) stage[j] = (j == 0) ? leftover : 0u;
        __syncwarp();
        gword += nwords;
        fill &= 31u;
    }
    if (lane == 0 && fill) {
        const uint32_t v = stage[0];
        if (v) atomicOr(&file_words[gword], v);
    }
}

// ------------------------------------------------------------------------------------------------
// K3b: Adler-32 combine.  State after row r: a' = a + S1_r, b' = b + n*a + S2_r  (mod 65521), start (1, 0).
// ------------------------------------------------------------------------------------------------
// ZLIB_AT: the file offset of the zlib stream (kPngEncHeaderSize for the files of png_encode_kernels.cu)
template <bool RAGGED = false, uint32_t ZLIB_AT = kPngHeaderSize>
__global__ void __launch_bounds__(kOffsetsThreads) adler_finalize_kernel(AdlerParams p)
{
    __shared__ unsigned long long s_red[3][kOffsetsThreads / 32];
    uint32_t img = blockIdx.x;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if constexpr (RAGGED) {                      // image blockIdx.x of p.desc (see row_offsets_kernel)
        const ImageDesc& d = p.desc[img];
        p.row_adler += d.row_base; p.st += img; p.out += d.out_ofs; p.w = d.w; p.h = d.h; p.chans = d.chans;
        img = 0;
    }
    const uint32_t h = p.h;
    unsigned long long s1 = 0, s2 = 0, wsum = 0;
    for (uint32_t y = tid; y < h; y += blockDim.x) {
        const uint2 v = p.row_adler[(size_t)img * h + y];
        s1 += v.x; s2 += v.y;
        wsum += (unsigned long long)((h - 1u - y) % kAdlerMod) * v.x;
        if ((y & 0xFFFFu) == 0xFFFFu) wsum %= kAdlerMod;
    }
    s1 = warp_sum_u64(s1); s2 = warp_sum_u64(s2); wsum = warp_sum_u64(wsum % kAdlerMod);
    if (lane == 0) { s_red[0][warp] = s1; s_red[1][warp] = s2; s_red[2][warp] = wsum; }
    __syncthreads();
    if (tid == 0) {
        unsigned long long S1 = 0, S2 = 0, W = 0;
        for (uint32_t i = 0; i < blockDim.x / 32; i++) { S1 += s_red[0][i]; S2 += s_red[1][i]; W += s_red[2][i]; }
        const unsigned long long n = ((unsigned long long)p.w * p.chans + 1ull) % kAdlerMod;
        const unsigned long long a = (1ull + S1) % kAdlerMod;
        const unsigned long long before = (h % kAdlerMod + W % kAdlerMod) % kAdlerMod;    // sum over rows of the running `a`
        const unsigned long long b = (S2 % kAdlerMod + n * before) % kAdlerMod;
        const uint32_t adler = (uint32_t)((b << 16) | a);
        const ImageState st = p.st[img];
        store_be32(p.out + (size_t)img * p.out_stride + ZLIB_AT + st.zsize - 4u, adler);
        p.st[img].adler = adler;
    }
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
template <int CHANS, int MODE>
static void launch_scan_t(const ScanParams& p, uint32_t n, bool hist, cudaStream_t s)
{
    dim3 grid((p.h + kRowsPerBlock - 1) / kRowsPerBlock, n);
    if (hist) row_scan_kernel<CHANS, MODE, true><<<grid, kScanThreads, 0, s>>>(p);
    else row_scan_kernel<CHANS, MODE, false><<<grid, kScanThreads, 0, s>>>(p);
}

void launch_scan(const ScanParams& p, uint32_t n, uint32_t chans, int mode, bool hist, cudaStream_t s)
{
    if (chans == 4) {
        if (mode == kLoadVec16) launch_scan_t<4, kLoadVec16>(p, n, hist, s);
        else if (mode == kLoadWords) launch_scan_t<4, kLoadWords>(p, n, hist, s);
        else launch_scan_t<4, kLoadBytes>(p, n, hist, s);
    } else {
        if (mode == kLoadWords) launch_scan_t<3, kLoadWords>(p, n, hist, s);
        else launch_scan_t<3, kLoadBytes>(p, n, hist, s);
    }
}

void launch_offsets(const OffsetsParams& p, uint32_t n, cudaStream_t s)
{
    row_offsets_kernel<false><<<n, kOffsetsThreads, 0, s>>>(p);
}

void launch_offsets_ragged(const OffsetsParams& p, uint32_t n, cudaStream_t s)
{
    row_offsets_kernel<true><<<n, kOffsetsThreads, 0, s>>>(p);
}

void launch_adler_finalize_ragged(const AdlerParams& p, uint32_t n, cudaStream_t s)
{
    adler_finalize_kernel<true><<<n, kOffsetsThreads, 0, s>>>(p);
}

void launch_adler_finalize_png(const AdlerParams& p, uint32_t n, cudaStream_t s)
{
    adler_finalize_kernel<true, kPngEncHeaderSize><<<n, kOffsetsThreads, 0, s>>>(p);
}

void launch_pack(const PackParams& p, uint32_t n, uint32_t chans, int mode, cudaStream_t s)
{
    dim3 grid((p.h + kRowsPerBlock - 1) / kRowsPerBlock, n);
    if (chans == 4) {
        if (mode == kLoadVec16) pack_rows_kernel<4, kLoadVec16><<<grid, kPackThreads, 0, s>>>(p);
        else if (mode == kLoadWords) pack_rows_kernel<4, kLoadWords><<<grid, kPackThreads, 0, s>>>(p);
        else pack_rows_kernel<4, kLoadBytes><<<grid, kPackThreads, 0, s>>>(p);
    } else {
        if (mode == kLoadWords) pack_rows_kernel<3, kLoadWords><<<grid, kPackThreads, 0, s>>>(p);
        else pack_rows_kernel<3, kLoadBytes><<<grid, kPackThreads, 0, s>>>(p);
    }
}

void launch_adler_finalize(const AdlerParams& p, uint32_t n, cudaStream_t s)
{
    adler_finalize_kernel<false><<<n, kOffsetsThreads, 0, s>>>(p);
}

}  // namespace fpngb
