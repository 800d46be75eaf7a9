// fpng_b200/csrc/decode_kernels.cu -- sm_90a kernels of the fpng decode hot path (fpng-written files only, like the
// reference: src/fpng.cpp:2209-2901).
//
// The reference decodes one serial Huffman bit-string (no row index exists in the format, SURVEY F6).  Here:
//   D1 decode_prepare_kernel   one warp per file: zlib/Deflate block header checks, code-length parse, fpng table
//                              constraints (fpng.cpp:1954-2076), 4096-entry literal/length LUT (fpng.cpp:1836-1895)
//   D2 decode_tokens_kernel    one CTA per file walks the stream in chunks of kDecThreads subsequences of kSubBits bits;
//                              inside a chunk every thread decodes its subsequence speculatively and the chunk iterates
//                              "restart at the predecessor's exit point" until no exit moves (self-synchronising prefix
//                              code; the first thread of a chunk always starts exactly), then a block scan of output byte
//                              counts places every subsequence in the filtered stream and a last decode writes the delta
//                              bytes (literals) / replicates the previous delta pixel (RLE matches, fpng.cpp:2289-2388)
//   D3 unfilter_kernel         inverse PNG filter 2 = running sum down each byte column (fpng.cpp:2439-2466 fuses it into
//                              the serial loop) + 24<->32bpp conversion (alpha 0xFF / dropped); for the *_typed calls
//                              unfilter_typed_kernel (decode_typed_kernels.cu) in the same slot, storing float / half / bf16
//   D2' decode_stored_kernel   stored-block files (fpng.cpp:2107-2207)
//   V2 decode_adler_kernel     opt-in (fpngb_set_decode_verify): zlib Adler-32 of the inflated stream from the delta rows
// Every stream violation the reference rejects ends in status FPNG_DECODE_NOT_FPNG (fpng.cpp:3131-3136).
#include "row_walk.cuh"
#include "kernels.cuh"
#include "decode.cuh"
#include "unfilter.cuh"

namespace fpngb {

__constant__ uint16_t c_len_base[32] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258, 0, 0, 0};
__constant__ uint8_t c_len_xbits[32] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0, 0, 0, 0};

// ------------------------------------------------------------------------------------------------
// bit reader over the zlib bytes of one file; reads past `limit` bytes return zero bits
// ------------------------------------------------------------------------------------------------
struct BitSrc {
    const uint8_t* z;          // zlib stream start (file + idat_ofs + 8), any alignment
    uint32_t limit;            // readable bytes from z (to the end of the file)
    __device__ __forceinline__ uint32_t word_at(uint32_t byte_ofs) const
    {
        // unaligned little-endian 32-bit read assembled from aligned words (z itself may be unaligned)
        const uintptr_t a = (uintptr_t)(z + byte_ofs);
        const uint32_t* p = (const uint32_t*)(a & ~(uintptr_t)3);
        const uint32_t sh = (uint32_t)(a & 3) * 8;
        uint32_t lo = 0, hi = 0;
        if (byte_ofs < limit) lo = __ldg(p);
        if (sh && byte_ofs + 4 - (sh >> 3) < limit) hi = __ldg(p + 1);
        uint32_t v = sh ? __funnelshift_r(lo, hi, sh) : lo;
        if (byte_ofs + 4 > limit) { const uint32_t valid = byte_ofs < limit ? limit - byte_ofs : 0; v &= valid >= 4 ? 0xFFFFFFFFu : ((1u << (8 * valid)) - 1u); }
        return v;
    }
};

struct BitCursor {
    unsigned long long buf; uint32_t cnt; uint32_t next_byte;   // next_byte: offset of the next unread byte
    unsigned long long pos;                                     // absolute bit position of buf's bit 0
    __device__ __forceinline__ void seek(const BitSrc& s, unsigned long long bitpos)
    {
        pos = bitpos;
        const uint32_t b = (uint32_t)(bitpos >> 3), sh = (uint32_t)(bitpos & 7);
        buf = ((unsigned long long)s.word_at(b) | ((unsigned long long)s.word_at(b + 4) << 32)) >> sh;
        cnt = 64 - sh; next_byte = b + 8;
    }
    __device__ __forceinline__ void refill(const BitSrc& s)
    {
        if (cnt <= 32) { buf |= (unsigned long long)s.word_at(next_byte) << cnt; cnt += 32; next_byte += 4; }
    }
    __device__ __forceinline__ uint32_t peek(uint32_t n) const { return (uint32_t)buf & ((1u << n) - 1u); }
    __device__ __forceinline__ void skip(uint32_t n) { buf >>= n; cnt -= n; pos += n; }
    __device__ __forceinline__ uint32_t get(const BitSrc& s, uint32_t n) { refill(s); const uint32_t v = peek(n); skip(n); return v; }
};

// ------------------------------------------------------------------------------------------------
// D1: per-file block header -> LUT
// ------------------------------------------------------------------------------------------------
// Canonical-code LUT with the reference's acceptance rule (fpng.cpp:1836-1895): complete code, or exactly one code.
// Runs on one warp; `sizes` in shared memory.
__device__ static bool build_lut_warp(const uint8_t* sizes, uint32_t nsyms, uint16_t* lut, uint32_t lut_bits, uint32_t lane, uint32_t* s_next /*17*/)
{
    __syncwarp();
    if (lane == 0) {
        uint32_t cnt[16];
        for (int i = 0; i < 16; i++) cnt[i] = 0;
        for (uint32_t i = 0; i < nsyms; i++) cnt[sizes[i]]++;
        uint32_t total = 0;
        s_next[0] = s_next[1] = 0;
        for (int l = 1; l <= 15; l++) { total = (total + cnt[l]) << 1; s_next[l + 1] = total; }
        uint32_t ok = 1;
        if (total != 0x10000u) {
            uint32_t used = 0;
            for (int l = 15; l >= 1; l--) used += cnt[l];
            ok = used == 1;
        }
        s_next[0] = ok;
    }
    __syncwarp();
    if (!s_next[0]) return false;
    const uint32_t lut_size = 1u << lut_bits;
    for (uint32_t i = lane; i < lut_size; i += 32) lut[i] = 0;
    __syncwarp();
    // canonical code of symbol i = first_code[len] + (number of earlier symbols of the same length); symbols are spread
    // over the lanes, each lane ranks and replicates its own
    for (uint32_t i = lane; i < nsyms; i += 32) {
        const uint32_t l = sizes[i];
        if (!l || l > lut_bits) continue;
        uint32_t rank = 0;
        for (uint32_t j = 0; j < i; j++) rank += sizes[j] == l;
        const uint32_t code = __brev(s_next[l] + rank) >> (32 - l);
        for (uint32_t c = code; c < lut_size; c += 1u << l) lut[c] = (uint16_t)(i | (l << 9));
    }
    __syncwarp();
    return true;
}

__global__ void __launch_bounds__(32) decode_prepare_kernel(DecodeParams p)
{
    __shared__ uint8_t s_sizes[288 + 32];
    __shared__ uint8_t s_cl[19];
    __shared__ uint16_t s_cllut[128];
    __shared__ uint32_t s_next[17];
    __shared__ uint32_t s_fail;
    __shared__ uint16_t s_base[4096];
    const uint32_t f = blockIdx.x, lane = threadIdx.x;
    const FileDesc fd = p.files[f];
    DecodeState* st = p.state + f;
    const uint8_t* z = p.d_files + fd.base + fd.idat_ofs + 8;
    BitSrc src{z, fd.file_size - (fd.idat_ofs + 8)};
    uint32_t* lut = p.luts + (size_t)f * 4096;

    if (lane == 0) {
        s_fail = 0;
        st->status = 0; st->stored = 0; st->token_start = 0; st->out_bytes = 0; st->end_byte = 0;
        // a file that failed before decoding (container walk, argument or shape checks): its bytes are never read
        if (fd.pre_status) s_fail = 1;
        // zlib header and block type (fpng.cpp:2219-2244)
        else if (fd.idat_len < 7 || z[0] != 0x78 || z[1] != 0x01) s_fail = 1;
        else if ((z[2] & 6) == 0) st->stored = 1;
        else if ((z[2] & 7) != 5) s_fail = 1;           // BFINAL = 1, BTYPE = 2
    }
    __syncwarp();
    if (s_fail) { if (lane == 0) st->status = 1; return; }
    if (st->stored) return;

    // HLIT / HDIST / HCLEN and the code-length code
    BitCursor bc; bc.seek(src, 16 + 3);
    const uint32_t nlit = bc.get(src, 5) + 257, ndist = bc.get(src, 5) + 1, nclen = bc.get(src, 4) + 4;
    if (lane < 19) s_cl[lane] = 0;
    __syncwarp();
    if (lane == 0) {
        const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
        for (uint32_t i = 0; i < nclen; i++) s_cl[order[i]] = (uint8_t)bc.get(src, 3);
    }
    __syncwarp();
    bool ok = nlit + ndist <= 288 + 32;
    ok = ok && build_lut_warp(s_cl, 19, s_cllut, 7, lane, s_next);
    if (!ok) { if (lane == 0) st->status = 1; return; }

    if (lane == 0) {
        for (uint32_t i = 0; i < 288 + 32; i++) s_sizes[i] = 0;
        uint32_t cur = 0, fail = 0;
        const uint32_t total = nlit + ndist;
        while (cur < total && !fail) {
            bc.refill(src);
            const uint32_t e = s_cllut[bc.peek(7)], l = e >> 9, s = e & 511;
            if (!l) { fail = 1; break; }
            bc.skip(l);
            if (s <= 15) { if (s > 12) { fail = 1; break; } s_sizes[cur++] = (uint8_t)s; continue; }   // fpng.cpp:2007
            uint32_t rep, val = 0;
            if (s == 16) { rep = bc.get(src, 2) + 3; if (!cur) { fail = 1; break; } val = s_sizes[cur - 1]; }
            else if (s == 17) rep = bc.get(src, 3) + 3;
            else rep = bc.get(src, 7) + 11;
            if (cur + rep > total) { fail = 1; break; }
            while (rep--) s_sizes[cur++] = (uint8_t)val;
        }
        // distance code constraints (fpng.cpp:2058-2074)
        uint32_t ones = 0;
        for (uint32_t i = 0; i < ndist && !fail; i++) ones += s_sizes[nlit + i] == 1;
        if (!fail) {
            if (ones < 1 || ones > 2) fail = 1;
            else if (s_sizes[nlit + fd.chans - 1] != 1) fail = 1;
            else if (ones == 2 && s_sizes[nlit + fd.chans] != 1) fail = 1;
        }
        for (uint32_t i = nlit; i < 288; i++) s_sizes[i] = 0;
        s_fail = fail;
        st->token_start = bc.pos;
    }
    __syncwarp();
    if (s_fail) { if (lane == 0) st->status = 1; return; }
    if (!build_lut_warp(s_sizes, 288, s_base, 12, lane, s_next)) { if (lane == 0) st->status = 1; return; }
    // Fuse a second literal into the entry when both codes fit in the 12 index bits (the reference augments its table the
    // same way, fpng.cpp:2079-2102):  sym0 | len0 << 9 | sym1 << 13 | len1 << 21.
    for (uint32_t i = lane; i < 4096; i += 32) {
        const uint32_t e0 = s_base[i], sym0 = e0 & 511u, len0 = e0 >> 9;
        uint32_t e = sym0 | (len0 << 9);
        if (len0 && sym0 < 256u) {
            const uint32_t e1 = s_base[i >> len0], sym1 = e1 & 511u, len1 = e1 >> 9;
            if (len1 && sym1 < 256u && len0 + len1 <= 12u) e |= (sym1 << 13) | (len1 << 21);
        }
        lut[i] = e;
    }
    // Fast table of the scan / write loops (one shared-memory look-up per 12 stream bits, one uniform code path):
    //   bits 0..3  L     stream bits consumed by the whole entry (0: not fast -- end of block, invalid code, a match whose
    //                    code + extra bits + distance bit do not fit in the 12 index bits; the loops fall back to `lut`)
    //   bits 4..5  cnt   number of literals (1..3), 0 = one match
    //   bits 8..31       the literals, first one in the low byte / the match's run length in bytes
    // followed by the 256 literal code sizes (the loops split a multi-literal entry at a subsequence boundary with them).
    uint32_t* fast = p.fast + (size_t)f * kFastWords;
    for (uint32_t i = lane; i < 4096; i += 32) {
        const uint32_t e0 = s_base[i], sym0 = e0 & 511u, len0 = e0 >> 9;
        uint32_t fe = 0;
        if (len0 && sym0 < 256u) {
            uint32_t L = len0, cnt = 1, P = sym0;
            for (uint32_t k = 1; k < 3; k++) {
                const uint32_t e1 = s_base[i >> L], sym1 = e1 & 511u, len1 = e1 >> 9;
                if (!len1 || sym1 >= 256u || L + len1 > 12u) break;
                P |= sym1 << (8u * k); L += len1; cnt++;
            }
            fe = L | (cnt << 4) | (P << 8);
        } else if (len0 && sym0 > 256u && sym0 <= 285u) {
            const uint32_t xb = c_len_xbits[sym0 - 257u];
            if (len0 + xb + 1u <= 12u) fe = (len0 + xb + 1u) | ((c_len_base[sym0 - 257u] + ((i >> len0) & ((1u << xb) - 1u))) << 8);
        }
        fast[i] = fe;
    }
    for (uint32_t i = lane; i < 64; i += 32)
        fast[4096 + i] = s_sizes[4 * i] | (s_sizes[4 * i + 1] << 8) | (s_sizes[4 * i + 2] << 16) | ((uint32_t)s_sizes[4 * i + 3] << 24);
}

// ------------------------------------------------------------------------------------------------
// D2: token decode.  The token bit-string of a file is cut into subsequences of kSubBits bits (absolute multiples of
// kSubBits in the aligned-stream bit coordinate).  Three kernels:
//   D2a decode_scan_kernel   one thread per subsequence, all files and subsequences in parallel: the thread starts
//                            p.pre_roll (kPreRoll) bits early (speculatively), lets the self-synchronising prefix code lock on, takes
//                            the first token boundary inside its subsequence as its start, then decodes to its exit (first
//                            boundary in the next subsequence) counting output bytes and remembering the last 4 literals.
//   D2b decode_link_kernel   one CTA per file walks the subsequences in order, 1024 at a time: verifies that every
//                            subsequence starts where its predecessor exits (the first one starts exactly, so a verified
//                            chain is the true parse), repairs the rare mismatches by re-decoding, and scans the byte
//                            counts / literal windows into the output offset and "previous pixel" of every subsequence.
//   D2c decode_write_kernel  one thread per live subsequence decodes again and writes the delta bytes.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kRelEnd = 0xFFFFFFFFu;              // exit flag (relative positions): saw the end-of-block code
constexpr uint32_t kRelErr = 0xFFFFFFFEu;              // exit flag: invalid code
constexpr unsigned long long kPosEnd = ~0ull;          // same flags in absolute (64-bit) form
constexpr unsigned long long kPosErr = ~0ull - 1;

// Aligned view of one file's zlib stream: 32-bit words starting at the 4-byte boundary at or before the stream.
struct Stream {
    const uint32_t* words;     // aligned base
    uint32_t max_widx;         // last readable word index (reads beyond are clamped: garbage but in bounds)
    uint32_t bit0;             // aligned-stream bit position of zlib bit 0 (0, 8, 16 or 24)
    // optional shared-memory window over words [sw_base, sw_base + sw_count): the scan and write kernels stage the 32 KiB of
    // stream their 256 subsequences walk (coalesced loads, one pad word per 32 so that threads 32 words apart hit different
    // banks); a refill is then a ~30-cycle shared load instead of an L1/L2 round trip in the middle of a dependent chain
    const uint32_t* swin; uint32_t sw_base, sw_count;
    __device__ __forceinline__ uint32_t word(uint32_t widx) const
    {
        const uint32_t si = widx - sw_base;
        if (si < sw_count) return swin[si + (si >> 5)];
        return __ldg(words + min(widx, max_widx));
    }
};
constexpr uint32_t kWinLead = 8, kWinTail = 8;                                   // words before / after the CTA's 256 subsequences
constexpr uint32_t kWinWords = kWinLead + kDecThreads * (kSubBits / 32) + kWinTail;
constexpr uint32_t kWinSmemWords = kWinWords + kWinWords / 32 + 1;

__device__ __forceinline__ void cp_async4(uint32_t* smem_dst, const uint32_t* gmem_src)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" :: "r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async16g(uint32_t* smem_dst, const uint32_t* gmem_src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" :: "r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src) : "memory");
}

// cooperative load of the CTA's stream window; `first_sub` = index of the CTA's first subsequence
__device__ __forceinline__ void stage_window(Stream& st, uint32_t* s_win, unsigned long long first_sub)
{
    const unsigned long long w0 = first_sub * (kSubBits / 32);
    const uint32_t base = (uint32_t)(w0 >= kWinLead ? w0 - kWinLead : 0ull);
    // word i lives at s_win[i + i / 32]; the pad slot in front of every 32-word block holds a COPY of the block's first word, so
    // that (address, address + 1) always are two consecutive stream words (win_peek below reads 32 bits at any bit position)
    // asynchronous copies (LDGSTS): all of a thread's ~33 words are in flight at once instead of one load -> store round trip each
    // (ncu: a quarter of the scan kernel's stall samples sat on the staging stores); the caller waits with stage_wait()
    for (uint32_t i = threadIdx.x; i < kWinWords; i += blockDim.x) {
        const uint32_t* src = st.words + min(base + i, st.max_widx);
        cp_async4(s_win + i + (i >> 5), src);
        if ((i & 31u) == 0u && i) cp_async4(s_win + i + (i >> 5) - 1u, src);
    }
    st.swin = s_win; st.sw_base = base; st.sw_count = kWinWords;
}

// the file's fast table (kFastWords words, 16-byte aligned) into shared memory, asynchronously
__device__ __forceinline__ void stage_fast_table(uint32_t* s_fast, const uint32_t* __restrict__ g_fast)
{
    for (uint32_t i = threadIdx.x; i < kFastWords / 4u; i += blockDim.x) cp_async16g(s_fast + 4u * i, g_fast + 4u * i);
}
__device__ __forceinline__ void stage_wait()
{
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;\n" ::: "memory");
    __syncthreads();
}

__device__ __forceinline__ Stream open_stream(const uint8_t* file, const FileDesc& fd)
{
    Stream st;
    const uint32_t zofs = fd.idat_ofs + 8;
    st.words = reinterpret_cast<const uint32_t*>(file + (zofs & ~3u));
    st.bit0 = (zofs & 3u) * 8u;
    st.max_widx = ((fd.file_size + 3u) >> 2) - 1u - (zofs >> 2);     // file buffers are padded to a multiple of 4
    st.swin = nullptr; st.sw_base = 0; st.sw_count = 0;
    return st;
}

struct Cursor {
    unsigned long long buf; uint32_t cnt, widx;
    uint32_t ahead;            // the next stream word, loaded one refill early so that its latency overlaps the decoding of ~32 bits
    __device__ __forceinline__ void seek(const Stream& st, unsigned long long abs_bit)
    {
        widx = (uint32_t)(abs_bit >> 5);
        const uint32_t sh = (uint32_t)abs_bit & 31u;
        const uint32_t lo = st.word(widx), hi = st.word(widx + 1u);
        buf = (((unsigned long long)hi << 32) | lo) >> sh;
        cnt = 64u - sh; widx += 2u;
        ahead = st.word(widx);
    }
    __device__ __forceinline__ void refill(const Stream& st)
    {
        if (cnt <= 32u) {
            buf |= (unsigned long long)ahead << cnt; cnt += 32u; widx++;
            ahead = st.word(widx);
        }
    }
    __device__ __forceinline__ void skip(uint32_t n) { buf >>= n; cnt -= n; }
};

struct SubScan {
    uint32_t first;      // rel. position of the first token boundary >= lo (the subsequence's start)
    uint32_t exit;       // rel. position of the first token boundary >= hi, or kRelEnd / kRelErr
    uint32_t eob_end;    // rel. position right after the EOB code (exit == kRelEnd)
    uint32_t n_out;      // bytes produced by tokens starting in [first, hi)
    uint32_t nlit;       // literal bytes among them (saturating at 255)
    uint32_t lits;       // last <= 4 literal bytes, most recent in the top byte
};

// Fused LUT entry: sym0 (9 bits) | len0 << 9 (4 bits) | sym1 << 13 (8 bits) | len1 << 21 (4 bits; 0 = no second literal)
__device__ __forceinline__ uint32_t lut_sym0(uint32_t e) { return e & 511u; }
__device__ __forceinline__ uint32_t lut_len0(uint32_t e) { return (e >> 9) & 15u; }
__device__ __forceinline__ uint32_t lut_sym1(uint32_t e) { return (e >> 13) & 255u; }
__device__ __forceinline__ uint32_t lut_len1(uint32_t e) { return e >> 21; }

// Write side of the token decoder: consecutive delta bytes of a row are combined into aligned 32-bit stores (the words
// a subsequence shares with its neighbours at either end, and row tails, go out as single bytes).
struct DeltaSink {
    uint8_t* delta; uint32_t pitch, bpl, h;
    uint32_t row, col;            // position in the filtered stream; col 0 is the filter byte
    uint8_t* ptr;                 // address of the next data byte of the current row
    uint32_t acc;                 // bytes [word(ptr), ptr) of the aligned word being filled, already in place
    uint32_t first_off;           // offset inside that word of the first byte this thread owns (0 unless it started mid-word)
    __device__ __forceinline__ void init(uint8_t* d, uint32_t pitch_, uint32_t bpl_, uint32_t h_, unsigned long long out_pos)
    {
        delta = d; pitch = pitch_; bpl = bpl_; h = h_;
        row = (uint32_t)(out_pos / (bpl + 1ull)); col = (uint32_t)(out_pos % (bpl + 1ull));
        ptr = delta + (size_t)row * pitch + (col ? col - 1u : 0u);
        acc = 0; first_off = (uint32_t)((uintptr_t)ptr & 3u);
    }
    // store the bytes gathered so far for the (incomplete or partly owned) current word, one by one
    __device__ __forceinline__ void flush()
    {
        const uint32_t n = (uint32_t)((uintptr_t)ptr & 3u);
        uint8_t* w = ptr - n;
        for (uint32_t i = first_off; i < n; i++) w[i] = (uint8_t)(acc >> (8u * i));
        acc = 0; first_off = n;
    }
    __device__ __forceinline__ void next_row() { flush(); col = 0; row++; ptr = delta + (size_t)row * pitch; first_off = 0; }
    // one data byte (col >= 1, row < h)
    __device__ __forceinline__ void put(uint32_t v)
    {
        acc |= v << (8u * ((uint32_t)(uintptr_t)ptr & 3u));
        ptr++;
        if (((uintptr_t)ptr & 3u) == 0) {                  // word complete
            if (first_off == 0) *reinterpret_cast<uint32_t*>(ptr - 4) = acc;
            else { for (uint32_t i = first_off; i < 4u; i++) ptr[(int)i - 4] = (uint8_t)(acc >> (8u * i)); first_off = 0; }
            acc = 0;
        }
        if (++col > bpl) next_row();
    }
};

// Decode from rel. position `rel` (origin = abs_origin bits in the aligned stream).  Tokens starting before `lo` are
// pre-roll (not counted); tokens starting in [lo, hi) are counted / written.  kWrite writes delta bytes.
template <bool kWrite>
__device__ __forceinline__ SubScan decode_range(const Stream& st, const uint32_t* __restrict__ s_lut, unsigned long long abs_origin,
                                                uint32_t rel, uint32_t lo, uint32_t hi, uint32_t chans,
                                                uint8_t* __restrict__ delta, uint32_t pitch, uint32_t bpl, uint32_t h,
                                                unsigned long long out_pos, uint32_t tail, uint32_t* err)
{
    SubScan r; r.first = lo; r.exit = 0; r.eob_end = 0; r.n_out = 0; r.nlit = 0; r.lits = 0;
    Cursor c; c.seek(st, abs_origin + rel);
    // ---- pre-roll: lock on to the token grid (speculative; an end-of-block or invalid code here means "not locked")
    while (rel < lo) {
        c.refill(st);
        const uint32_t e = s_lut[(uint32_t)c.buf & 4095u];
        uint32_t l = lut_len0(e);
        const uint32_t s = lut_sym0(e);
        if (!l || s == 256u || s > 285u) { rel = lo; c.seek(st, abs_origin + rel); break; }
        if (s > 256u) { const uint32_t xb = c_len_xbits[s - 257u]; l += xb + 1u; }
        c.skip(l); rel += l;
    }
    r.first = rel;
    uint32_t lits = tail;
    DeltaSink sink;
    if (kWrite) sink.init(delta, pitch, bpl, h, out_pos);
    uint32_t n_out = 0, nlit = 0;
    while (rel < hi) {
        c.refill(st);
        const uint32_t e = s_lut[(uint32_t)c.buf & 4095u];
        const uint32_t l0 = lut_len0(e), s = lut_sym0(e);
        if (!l0) { r.exit = kRelErr; r.n_out = n_out; r.nlit = nlit; r.lits = lits; return r; }
        if (s < 256u) {
            // one literal, or two when the fused second literal also starts inside the subsequence
            const uint32_t l1 = lut_len1(e);
            const bool two = l1 && (rel + l0 < hi);
            const uint32_t l = two ? l0 + l1 : l0;
            c.skip(l); rel += l;
            const uint32_t cntl = two ? 2u : 1u;
            n_out += cntl; nlit += cntl;
            if (!kWrite) {
                lits = (lits >> 8) | (s << 24);
                if (two) lits = (lits >> 8) | (lut_sym1(e) << 24);
            } else {
                // first literal, then (predicated) the fused second one; a literal at column 0 is the row's filter byte
                lits = (lits >> 8) | (s << 24);
                if (sink.col == 0) { if (sink.row >= h || s != (sink.row ? 2u : 0u)) { *err = 1; break; } sink.col = 1; }   // fpng.cpp:2264, 2642
                else sink.put(s);
                if (two) {
                    const uint32_t v = lut_sym1(e);
                    lits = (lits >> 8) | (v << 24);
                    if (sink.col == 0) { if (sink.row >= h || v != (sink.row ? 2u : 0u)) { *err = 1; break; } sink.col = 1; }
                    else sink.put(v);
                }
            }
        } else if (s == 256u) {
            c.skip(l0); rel += l0;
            if (kWrite) sink.flush();
            r.exit = kRelEnd; r.eob_end = rel; r.n_out = n_out; r.nlit = nlit; r.lits = lits;
            return r;
        } else {
            if (s > 285u) { r.exit = kRelErr; r.n_out = n_out; r.nlit = nlit; r.lits = lits; return r; }
            c.skip(l0);
            const uint32_t xb = c_len_xbits[s - 257u];
            const uint32_t run = c_len_base[s - 257u] + ((uint32_t)c.buf & ((1u << xb) - 1u));
            c.skip(xb + 1u);                                                       // extra bits + the 1-bit distance code (fpng.cpp:2300)
            rel += l0 + xb + 1u;
            n_out += run;
            if (kWrite) {
                // run of the previous delta pixel: starts on a pixel boundary after at least one pixel of the row, is a
                // whole number of pixels and stays inside the row (fpng.cpp:2302-2315, 2681-2691, 2727)
                const uint32_t row = sink.row, col = sink.col;
                const bool bad = row >= h || col < 1u + chans || ((col - 1u) % chans) != 0 || (run % chans) != 0 || (col - 1u) + run > bpl;
                if (bad) { *err = 1; return r; }
                const uint32_t px = chans == 4 ? lits : (lits >> 8);              // last `chans` literals, oldest in the low byte
                if (chans == 4) {
                    // RGBA pixels are word aligned in the delta rows: one 32-bit store per pixel
                    sink.flush();
                    uint32_t* d = reinterpret_cast<uint32_t*>(sink.ptr);
                    const uint32_t npx = run >> 2;
                    for (uint32_t i = 0; i < npx; i++) d[i] = px;
                    sink.ptr += run; sink.col += run;
                    if (sink.col > bpl) sink.next_row();
                } else {
                    for (uint32_t i = 0; i < run; i += 3) { sink.put(px & 0xFFu); sink.put((px >> 8) & 0xFFu); sink.put(px >> 16); }
                }
            }
        }
    }
    if (kWrite) sink.flush();
    r.exit = rel; r.n_out = n_out; r.nlit = nlit; r.lits = lits;
    return r;
}

// Write pass, lean form: decodes the tokens of one subsequence from its verified start and stores the delta bytes.
// Output state is three 32-bit values (row, data column, pending-byte accumulator) and a row pointer; bytes are gathered into
// aligned 32-bit stores (a thread's unaligned head bytes and a row's tail bytes go out singly, so neighbouring threads
// never touch the same word).  Same acceptance rules as decode_range<true> (fpng.cpp:2264, 2302-2315, 2642, 2681-2691, 2727).
// ---- lean token loops on the shared-memory window -------------------------------------------------------------------
// With the stream staged in shared memory a decoder needs no bit buffer: 32 fresh bits at ANY bit position are two shared
// loads and one funnel shift, and the only state carried from token to token is the bit position itself.
__device__ __forceinline__ uint32_t win_peek(const uint32_t* __restrict__ win, uint32_t q)     // q: bit offset from the window's first word
{
    const uint32_t si = q >> 5, a = si + (si >> 5);
    return __funnelshift_r(win[a], win[a + 1u], q);                         // shift amount taken modulo 32
}

// One step of the fast loops: looks up the entry at bit position q of the window.  A multi-literal entry whose later
// literals could start at or beyond `limit` (the subsequence boundary) is cut down to its first literal.  Returns false when
// the entry is not fast (L = 0); then `w` still holds the 32 stream bits for the fall-back.
struct FastTok { uint32_t L, cnt, payload, w; };
__device__ __forceinline__ bool fast_tok(const uint32_t* __restrict__ win, const uint32_t* __restrict__ s_fast, uint32_t sizes_s, uint32_t q, uint32_t rel, uint32_t limit, FastTok& t)
{
    t.w = win_peek(win, q);
    const uint32_t e = s_fast[t.w & 4095u];
    t.L = e & 15u; t.cnt = (e >> 4) & 3u; t.payload = e >> 8;
    if (t.cnt >= 2u && rel + 12u > limit) {
        t.payload &= 0xFFu; t.cnt = 1u;
        asm("ld.shared.u8 %0, [%1];\n" : "=r"(t.L) : "r"(sizes_s + t.payload));      // code size of the first literal
    }
    return t.L != 0u;
}

// Fall-back of the fast loops: one token through the single-token table in global memory.  Returns the token's length in bits
// (0 = invalid code), sets sym (256 = end of block) and, for a match, run.
__device__ __forceinline__ uint32_t slow_tok(const uint32_t* __restrict__ lutg, uint32_t w, uint32_t& sym, uint32_t& run)
{
    const uint32_t e = __ldg(lutg + (w & 4095u));
    const uint32_t l0 = lut_len0(e);
    sym = lut_sym0(e); run = 0;
    if (!l0 || sym > 285u) return 0u;
    if (sym <= 256u) return l0;
    const uint32_t xb = c_len_xbits[sym - 257u];
    run = c_len_base[sym - 257u] + ((w >> l0) & ((1u << xb) - 1u));
    return l0 + xb + 1u;                                                     // extra bits + the 1-bit distance code (fpng.cpp:2300)
}

// Scan pass on the window: same contract as decode_range<false>.  `O` = bit offset of abs_origin inside the window.
__device__ __forceinline__ SubScan scan_window(const uint32_t* __restrict__ win, uint32_t O, const uint32_t* __restrict__ s_fast,
                                               const uint32_t* __restrict__ lutg, uint32_t rel, uint32_t lo, uint32_t hi)
{
    SubScan r; r.first = lo; r.exit = 0; r.eob_end = 0; r.n_out = 0; r.nlit = 0; r.lits = 0;
    FastTok t;
    const uint32_t sizes_s = (uint32_t)__cvta_generic_to_shared(s_fast + 4096);
    while (rel < lo) {                                                       // pre-roll: lock on to the token grid
        if (fast_tok(win, s_fast, sizes_s, O + rel, rel, lo, t)) { rel += t.L; continue; }
        uint32_t sym, run;
        const uint32_t l = slow_tok(lutg, t.w, sym, run);
        if (!l || sym == 256u) { rel = lo; break; }                          // not locked on
        rel += l;
    }
    r.first = rel;
    uint32_t lits = 0, n_out = 0, nlit = 0;
    while (rel < hi) {
        if (fast_tok(win, s_fast, sizes_s, O + rel, rel, hi, t)) {
            rel += t.L;
            n_out += t.cnt ? t.cnt : t.payload;
            nlit += t.cnt;
            lits = __funnelshift_r(lits, t.payload, 8u * t.cnt);              // the new literals enter at the top (cnt = 0: unchanged)
            continue;
        }
        uint32_t sym, run;
        const uint32_t l = slow_tok(lutg, t.w, sym, run);
        if (!l) { r.exit = kRelErr; r.n_out = n_out; r.nlit = nlit; r.lits = lits; return r; }
        rel += l;
        if (sym == 256u) { r.exit = kRelEnd; r.eob_end = rel; r.n_out = n_out; r.nlit = nlit; r.lits = lits; return r; }
        if (sym < 256u) { n_out++; nlit++; lits = (lits >> 8) | (sym << 24); }   // (cannot happen: every literal is a fast entry)
        else n_out += run;
    }
    r.exit = rel; r.n_out = n_out; r.nlit = nlit; r.lits = lits;
    return r;
}

template <int CHANS>
__device__ __forceinline__ void decode_write_range(const Stream& st, const uint32_t* __restrict__ s_fast, const uint32_t* __restrict__ lutg, unsigned long long abs_origin, uint32_t hi,
                                                   uint8_t* __restrict__ delta, uint32_t pitch, uint32_t bpl, uint32_t h,
                                                   unsigned long long out_pos, uint32_t tail, uint32_t* err)
{
    // the subsequence lies inside the CTA's shared-memory window (stage_window): read it by bit position
    const uint32_t* __restrict__ win = st.swin;
    const uint32_t O = (uint32_t)(abs_origin - 32ull * st.sw_base);
    uint32_t rel = 0, lits = tail;
    uint32_t row = (uint32_t)(out_pos / (bpl + 1ull));
    const uint32_t col0 = (uint32_t)(out_pos % (bpl + 1ull));
    bool need_filter = col0 == 0u;                     // the next byte of the filtered stream is the row's filter byte
    uint32_t dcol = col0 ? col0 - 1u : 0u;             // data bytes of the current row already produced
    uint8_t* rowp = delta + (size_t)row * pitch;
    unsigned long long acc = 0; uint32_t nacc = 0;     // pending bytes: data columns [dcol - nacc, dcol), first one 4-byte aligned
    // Completed words of the literal fast path wait in a 4-deep register queue (newest in q3) and leave as ONE 128-bit store once
    // they fill a 16-byte aligned group: the write pass is bound by store transactions (every lane writes its own region, so a
    // 32-bit store costs a whole L1 tag cycle per lane), not by decoding.  Every other path flushes the queue first.
    uint32_t q0 = 0, q1 = 0, q2 = 0, q3 = 0, nq = 0;   // queued words: data columns [dcol - nacc - 4 nq, dcol - nacc)
#define FPNGB_FLUSHQ() do { \
        if (nq) { \
            uint32_t* b__ = reinterpret_cast<uint32_t*>(rowp + dcol - nacc - 4u * nq); \
            if (nq == 3u) { b__[0] = q1; b__[1] = q2; b__[2] = q3; } \
            else if (nq == 2u) { b__[0] = q2; b__[1] = q3; } \
            else b__[0] = q3; \
            nq = 0u; \
        } \
    } while (0)

    // general byte sink: unaligned head bytes of the thread's range and a scanline's last bytes go out singly, everything else
    // as aligned 32-bit words
#define FPNGB_EMIT(v) do { \
        const uint32_t v__ = (v); \
        if (nacc == 0u && (dcol & 3u)) rowp[dcol] = (uint8_t)v__; \
        else { acc |= (unsigned long long)v__ << (8u * nacc); if (++nacc == 4u) { *reinterpret_cast<uint32_t*>(rowp + dcol - 3u) = (uint32_t)acc; acc = 0ull; nacc = 0u; } } \
        if (++dcol == bpl) { \
            for (uint32_t i__ = 0; i__ < nacc; i__++) rowp[dcol - nacc + i__] = (uint8_t)(acc >> (8u * i__)); \
            acc = 0ull; nacc = 0u; row++; rowp += pitch; dcol = 0u; need_filter = true; \
        } \
    } while (0)
#define FPNGB_LITERAL(v) do { \
        const uint32_t s__ = (v); \
        lits = (lits >> 8) | (s__ << 24); \
        if (need_filter) { if (row >= h || s__ != (row ? 2u : 0u)) { *err = 1; return; } need_filter = false; } \
        else { if (row >= h) { *err = 1; return; } FPNGB_EMIT(s__); } \
    } while (0)

    // literal fast path allowed: inside a scanline (filter byte consumed, row valid) with the pending bytes word aligned; the fast path
    // itself keeps this true, every other path re-evaluates it when it is done
    bool fastok;
#define FPNGB_REFLAG() (fastok = !need_filter && row < h && (nacc | ((dcol & 3u) == 0u)))
    FPNGB_REFLAG();
    FastTok t;
    const uint32_t sizes_s = (uint32_t)__cvta_generic_to_shared(s_fast + 4096);
    while (rel < hi) {
        uint32_t run;
        if (fast_tok(win, s_fast, sizes_s, O + rel, rel, hi, t)) {
            rel += t.L;
            if (t.cnt) {
                const uint32_t cnt = t.cnt, P = t.payload;
                // fast path (almost every literal): inside a scanline, the pending bytes word aligned -- append the one to three bytes
                // to the 64-bit accumulator, store a word when four are there; no per-byte branches
                if (fastok && dcol + cnt < bpl) {
                    lits = __funnelshift_r(lits, P, 8u * cnt);
                    acc |= (unsigned long long)P << (8u * nacc);
                    nacc += cnt; dcol += cnt;
                    if (nacc >= 4u) {
                        const uint32_t wv = (uint32_t)acc;
                        acc >>= 32; nacc -= 4u;
                        const uint32_t wcol = dcol - nacc - 4u;              // data column of this word
                        if (nq == 0u && (wcol & 15u)) *reinterpret_cast<uint32_t*>(rowp + wcol) = wv;   // not yet at a 16-byte boundary
                        else {
                            q0 = q1; q1 = q2; q2 = q3; q3 = wv;
                            if (++nq == 4u) { *reinterpret_cast<uint4*>(rowp + wcol - 12u) = make_uint4(q0, q1, q2, q3); nq = 0u; }
                        }
                    }
                    continue;
                }
                FPNGB_FLUSHQ();
                FPNGB_LITERAL(P & 0xFFu);
                if (cnt > 1u) FPNGB_LITERAL((P >> 8) & 0xFFu);
                if (cnt > 2u) FPNGB_LITERAL(P >> 16);
                FPNGB_REFLAG();
                continue;
            }
            run = t.payload;
        } else {
            uint32_t sym;
            const uint32_t l = slow_tok(lutg, t.w, sym, run);
            if (!l) return;                                                // invalid code: the link pass already flagged it
            if (sym == 256u) break;
            rel += l;
            if (sym < 256u) { FPNGB_FLUSHQ(); FPNGB_LITERAL(sym); FPNGB_REFLAG(); continue; }
        }
        {
            FPNGB_FLUSHQ();
            const bool bad = row >= h || need_filter || dcol < (uint32_t)CHANS || (dcol % CHANS) != 0u || (run % CHANS) != 0u || dcol + run > bpl;
            if (bad) { *err = 1; return; }
            const uint32_t px = CHANS == 4 ? lits : (lits >> 8);          // last CHANS literals, oldest in the low byte
            if (CHANS == 4) {
                // dcol % 4 == 0: nothing is pending, pixels are word aligned
                uint32_t* d = reinterpret_cast<uint32_t*>(rowp + dcol);
                const uint32_t npx = run >> 2;
                uint32_t i = 0;
                for (; i < npx && ((dcol + 4u * i) & 15u); i++) d[i] = px;             // up to the next 16-byte boundary
                const uint4 px4 = make_uint4(px, px, px, px);
                for (; i + 4u <= npx; i += 4u) *reinterpret_cast<uint4*>(d + i) = px4;
                for (; i < npx; i++) d[i] = px;
                dcol += run;
                if (dcol == bpl) { row++; rowp += pitch; dcol = 0u; need_filter = true; }
            } else {
                // RGB: the 3-byte pixel repeats with a period of three 32-bit words.  Bytes up to the next word boundary go through
                // the byte sink, whole words are stored from three rotating pattern registers, the remainder again byte-wise.
                uint32_t left = run, ph = 0;                                  // ph: index inside the pixel of the next byte
                while (left && ((dcol & 3u) || nacc)) { FPNGB_EMIT((px >> (8u * ph)) & 0xFFu); ph = ph == 2u ? 0u : ph + 1u; left--; }
                if (left >= 4u) {
                    uint32_t wa = 0, wb = 0, wc = 0;
#pragma unroll
                    for (uint32_t j = 0; j < 4; j++) {
                        wa |= ((px >> (8u * ((ph + j) % 3u))) & 0xFFu) << (8u * j);
                        wb |= ((px >> (8u * ((ph + 4u + j) % 3u))) & 0xFFu) << (8u * j);
                        wc |= ((px >> (8u * ((ph + 8u + j) % 3u))) & 0xFFu) << (8u * j);
                    }
                    const uint32_t nwords = left >> 2;
                    uint32_t* d = reinterpret_cast<uint32_t*>(rowp + dcol);
                    uint32_t k = 0;
                    for (; k < nwords && ((dcol + 4u * k) & 15u); k++) { d[k] = wa; const uint32_t tw = wa; wa = wb; wb = wc; wc = tw; }
                    for (; k + 4u <= nwords; k += 4u) {                       // four words advance the 3-word pattern by one
                        *reinterpret_cast<uint4*>(d + k) = make_uint4(wa, wb, wc, wa);
                        const uint32_t tw = wa; wa = wb; wb = wc; wc = tw;
                    }
                    for (; k < nwords; k++) { d[k] = wa; const uint32_t tw = wa; wa = wb; wb = wc; wc = tw; }
                    dcol += nwords << 2; left -= nwords << 2; ph = (ph + nwords) % 3u;      // 4 bytes advance the phase by 1
                    if (dcol == bpl) { row++; rowp += pitch; dcol = 0u; need_filter = true; }   // a run may end exactly at the end of its scanline
                }
                while (left) { FPNGB_EMIT((px >> (8u * ph)) & 0xFFu); ph = ph == 2u ? 0u : ph + 1u; left--; }
            }
            FPNGB_REFLAG();
        }
    }
    FPNGB_FLUSHQ();
    for (uint32_t i = 0; i < nacc; i++) rowp[dcol - nacc + i] = (uint8_t)(acc >> (8u * i));
#undef FPNGB_FLUSHQ
#undef FPNGB_REFLAG
#undef FPNGB_EMIT
#undef FPNGB_LITERAL
}

// "keep the last 4 literal bytes" monoid: a then b  (v holds the last n literals, most recent in the top byte)
__device__ __forceinline__ void lit_combine(uint32_t& n, uint32_t& v, uint32_t nb, uint32_t vb)
{
    if (nb >= 4u) { n = 4u; v = vb; return; }
    if (nb == 0u) return;
    v = (v >> (8u * nb)) | (vb & (0xFFFFFFFFu << (8u * (4u - nb))));
    n = min(n + nb, 4u);
}

// subsequence g of a file covers aligned-stream bits [g*kSubBits, (g+1)*kSubBits)
struct FileSpan { unsigned long long tok0; unsigned long long g0, g1; };     // first token bit; first/last subsequence index
__device__ __forceinline__ FileSpan file_span(const DecodeState& st, const Stream& sm, const FileDesc& fd)
{
    FileSpan f;
    f.tok0 = st.token_start + sm.bit0;
    const unsigned long long endbit = (unsigned long long)(fd.idat_len > 4u ? fd.idat_len - 4u : 0u) * 8ull + sm.bit0;   // tokens (and EOB) end before the Adler bytes
    f.g0 = f.tok0 / kSubBits;
    f.g1 = endbit ? (endbit - 1ull) / kSubBits : 0ull;
    if (f.g1 < f.g0) f.g1 = f.g0;
    return f;
}

__global__ void __launch_bounds__(kDecThreads) decode_scan_kernel(DecodeParams p)
{
    extern __shared__ __align__(16) uint32_t dec_smem[];
    uint32_t* s_fast = dec_smem;                      // [kFastWords]
    uint32_t* s_win = dec_smem + kFastWords;          // [kWinSmemWords]
    const uint32_t f = blockIdx.y, tid = threadIdx.x;
    const DecodeState st = p.state[f];
    if (st.status || st.stored) return;
    const FileDesc fd = p.files[f];
    Stream sm = open_stream(p.d_files + fd.base, fd);
    const FileSpan sp = file_span(st, sm, fd);
    const unsigned long long g = sp.g0 + (unsigned long long)blockIdx.x * kDecThreads + tid;
    if (sp.g0 + (unsigned long long)blockIdx.x * kDecThreads > sp.g1) return;
    stage_fast_table(s_fast, p.fast + (size_t)f * kFastWords);
    stage_window(sm, s_win, sp.g0 + (unsigned long long)blockIdx.x * kDecThreads);
    stage_wait();
    if (g > sp.g1) return;
    const uint32_t* lutg = p.luts + (size_t)f * 4096;
    SubInfo* info = p.subs + fd.sub_base + (g - sp.g0);
    const unsigned long long lo_abs = g * kSubBits;
    SubScan r;
    unsigned long long origin;
    if (g == sp.g0) {            // the file's first subsequence starts exactly at the first token
        origin = sp.tok0;
        r = scan_window(s_win, (uint32_t)(origin - 32ull * sm.sw_base), s_fast, lutg, 0u, 0u, (uint32_t)((g + 1) * kSubBits - origin));
    } else {
        origin = lo_abs < sp.tok0 + p.pre_roll ? sp.tok0 : lo_abs - p.pre_roll;   // never pre-roll across the block header
        r = scan_window(s_win, (uint32_t)(origin - 32ull * sm.sw_base), s_fast, lutg, 0u, (uint32_t)(lo_abs - origin), (uint32_t)(lo_abs - origin) + kSubBits);
    }
    info->start = origin + r.first;
    info->exit = r.exit >= kRelErr ? (r.exit == kRelEnd ? kPosEnd : kPosErr) : origin + r.exit;
    info->eob_end = origin + r.eob_end;
    info->n_out = r.n_out; info->lits = r.lits; info->nlit = min(r.nlit, 4u);
}

// statistics: subsequences whose speculative start was wrong and had to be decoded again by the link pass (fpngb_debug_decode_repairs)
__device__ unsigned long long g_link_repairs = 0ull;
unsigned long long decode_link_repairs(bool reset)
{
    unsigned long long v = 0, z = 0;
    cudaMemcpyFromSymbol(&v, g_link_repairs, sizeof v);
    if (reset) cudaMemcpyToSymbol(g_link_repairs, &z, sizeof z);
    return v;
}

__global__ void __launch_bounds__(kLinkThreads) decode_link_kernel(DecodeParams p)
{
    __shared__ uint32_t s_lut[4096];
    __shared__ unsigned long long s_exit[kLinkThreads];
    __shared__ unsigned long long s_scan[kLinkThreads / 32];
    __shared__ uint32_t s_litn[kLinkThreads / 32], s_litv[kLinkThreads / 32];
    __shared__ unsigned long long s_wbase[kLinkThreads / 32], s_chunk_total;
    __shared__ uint32_t s_wlitn[kLinkThreads / 32], s_wlitv[kLinkThreads / 32], s_chunk_litn, s_chunk_litv;
    __shared__ unsigned long long s_carry_start, s_carry_out, s_eob_end;
    __shared__ uint32_t s_carry_litn, s_carry_litv, s_done, s_err, s_first_bad, s_lut_loaded;

    const uint32_t f = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    DecodeState* stp = p.state + f;
    if (stp->status || stp->stored) return;
    const DecodeState st = *stp;
    const FileDesc fd = p.files[f];
    const Stream sm = open_stream(p.d_files + fd.base, fd);
    const FileSpan sp = file_span(st, sm, fd);
    const uint32_t chans = fd.chans, bpl = fd.w * chans, h = fd.h;
    const unsigned long long total_out = (unsigned long long)(bpl + 1) * h;
    SubInfo* subs = p.subs + fd.sub_base;
    const unsigned long long nsub = sp.g1 - sp.g0 + 1ull;

    if (tid == 0) { s_carry_start = sp.tok0; s_carry_out = 0; s_carry_litn = 0; s_carry_litv = 0; s_done = 0; s_err = 0; s_eob_end = 0; s_lut_loaded = 0; }
    __syncthreads();

    SubInfo nxt;                                       // the next chunk's records are loaded while this chunk is processed
    if (tid < nsub) nxt = subs[tid];
    for (unsigned long long base = 0; base < nsub; base += kLinkThreads) {
        const unsigned long long i = base + tid;
        const bool have = i < nsub;
        SubInfo in;
        if (have) in = nxt;
        else { in.start = 0; in.exit = kPosErr; in.eob_end = 0; in.n_out = 0; in.lits = 0; in.nlit = 0; }
        if (i + kLinkThreads < nsub) nxt = subs[i + kLinkThreads];
        const unsigned long long g = sp.g0 + i;
        // ---- verify / repair the chain: every subsequence must start where its predecessor exits
        for (uint32_t iter = 0;; iter++) {
            s_exit[tid] = in.exit;
            __syncthreads();
            const unsigned long long want = tid == 0 ? s_carry_start : s_exit[tid - 1];
            const int mismatch = have && want < kPosErr && want != in.start;
            if (!__syncthreads_or(mismatch)) break;
            if (!s_lut_loaded) {                       // repairs are rare: fetch the LUT only when first needed
                for (uint32_t k = tid; k < 4096; k += blockDim.x) s_lut[k] = p.luts[(size_t)f * 4096 + k];
                __syncthreads();
                if (tid == 0) s_lut_loaded = 1;
            }
            if (mismatch) {
                atomicAdd(&g_link_repairs, 1ull);
                const unsigned long long hi_abs = (g + 1) * kSubBits;
                if (want >= hi_abs) { in.start = want; in.exit = want; in.n_out = 0; in.nlit = 0; in.lits = 0; }   // cannot happen for kSubBits >> token size
                else {
                    const SubScan r = decode_range<false>(sm, s_lut, want, 0u, 0u, (uint32_t)(hi_abs - want), chans, nullptr, 0, 0, 0, 0, 0, nullptr);
                    in.start = want;
                    in.exit = r.exit >= kRelErr ? (r.exit == kRelEnd ? kPosEnd : kPosErr) : want + r.exit;
                    in.eob_end = want + r.eob_end; in.n_out = r.n_out; in.lits = r.lits; in.nlit = min(r.nlit, 4u);
                }
            }
            __syncthreads();
        }
        // the first subsequence that ends in EOB / an invalid code terminates the stream; everything after it is dead
        if (tid == 0) s_first_bad = kLinkThreads;
        __syncthreads();
        if (in.exit >= kPosErr) atomicMin(&s_first_bad, tid);
        __syncthreads();
        const uint32_t first_bad = s_first_bad;
        const bool live = have && tid <= first_bad;
        if (!live) { in.n_out = 0; in.nlit = 0; in.lits = 0; }

        // ---- block-exclusive scans: output byte offset and literal window entering each subsequence
        unsigned long long incl = in.n_out;
        uint32_t wn = in.nlit, wv = in.lits;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long up = __shfl_up_sync(kFullMask, incl, o);
            const uint32_t un = __shfl_up_sync(kFullMask, wn, o), uv = __shfl_up_sync(kFullMask, wv, o);
            if (lane >= (uint32_t)o) { incl += up; uint32_t tn = un, tv = uv; lit_combine(tn, tv, wn, wv); wn = tn; wv = tv; }
        }
        if (lane == 31) { s_scan[warp] = incl; s_litn[warp] = wn; s_litv[warp] = wv; }
        unsigned long long ex = __shfl_up_sync(kFullMask, incl, 1);
        uint32_t en = __shfl_up_sync(kFullMask, wn, 1), ev = __shfl_up_sync(kFullMask, wv, 1);
        if (lane == 0) { ex = 0; en = 0; ev = 0; }
        __syncthreads();
        // second level: warp 0 scans the (<= 32) warp totals, carry of the earlier chunks folded in
        static_assert(kLinkThreads / 32 <= 32, "one warp scans the warp totals");
        if (warp == 0) {
            const bool hw = lane < kLinkThreads / 32;
            unsigned long long t = hw ? s_scan[lane] : 0ull;
            uint32_t tn = hw ? s_litn[lane] : 0u, tv = hw ? s_litv[lane] : 0u;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned long long up = __shfl_up_sync(kFullMask, t, o);
                const uint32_t un = __shfl_up_sync(kFullMask, tn, o), uv = __shfl_up_sync(kFullMask, tv, o);
                if (lane >= (uint32_t)o) { t += up; uint32_t an = un, av = uv; lit_combine(an, av, tn, tv); tn = an; tv = av; }
            }
            // exclusive form, then the carry in front
            unsigned long long xt = __shfl_up_sync(kFullMask, t, 1);
            uint32_t xn = __shfl_up_sync(kFullMask, tn, 1), xv = __shfl_up_sync(kFullMask, tv, 1);
            if (lane == 0) { xt = 0; xn = 0; xv = 0; }
            uint32_t bn0 = s_carry_litn, bv0 = s_carry_litv;
            lit_combine(bn0, bv0, xn, xv);
            if (hw) { s_wbase[lane] = xt; s_wlitn[lane] = bn0; s_wlitv[lane] = bv0; }
            if (lane == 31) {                                             // lanes beyond the last warp carry zeros: lane 31 holds the chunk totals
                uint32_t cn0 = s_carry_litn, cv0 = s_carry_litv;
                lit_combine(cn0, cv0, tn, tv);
                s_chunk_total = t; s_chunk_litn = cn0; s_chunk_litv = cv0;
            }
        }
        __syncthreads();
        const unsigned long long wbase = s_wbase[warp], chunk_total = s_chunk_total;
        uint32_t bn = s_wlitn[warp], bv = s_wlitv[warp];
        const uint32_t cn = s_chunk_litn, cv = s_chunk_litv;
        lit_combine(bn, bv, en, ev);
        const unsigned long long out_pos = s_carry_out + wbase + ex;

        if (have) {
            SubInfo o;
            o.start = in.start; o.exit = out_pos; o.eob_end = 0; o.n_out = live ? in.n_out : 0u; o.lits = bv; o.nlit = live ? 1u : 0u;
            if (live && out_pos + in.n_out > total_out) { o.n_out = 0; o.nlit = 0; s_err = 1; }
            subs[i] = o;
        }
        if (have && tid == first_bad) { if (in.exit == kPosEnd) { s_eob_end = in.eob_end; s_done = 1; } else s_err = 1; }
        __syncthreads();
        if (tid == 0) {
            s_carry_start = s_exit[kLinkThreads - 1];
            s_carry_out += chunk_total; s_carry_litn = cn; s_carry_litv = cv;
            if (s_carry_out > total_out) s_err = 1;
        }
        __syncthreads();
        if (s_done || s_err) {
            // mark the remaining subsequences dead so the write kernel skips them
            for (unsigned long long k = base + kLinkThreads + tid; k < nsub; k += kLinkThreads) { subs[k].n_out = 0; subs[k].nlit = 0; }
            break;
        }
    }
    __syncthreads();
    if (tid == 0) {
        // EOB right after the last row, then pad to a byte, then exactly the 4 Adler bytes (fpng.cpp:2559-2584)
        const unsigned long long used = s_eob_end >= sm.bit0 ? ((s_eob_end - sm.bit0 + 7ull) >> 3) : 0ull;
        const bool ok = !s_err && s_done && s_carry_out == total_out && used + 4ull == fd.idat_len;
        stp->status = ok ? 0u : 1u;
        stp->out_bytes = s_carry_out; stp->end_byte = used;
    }
}

__global__ void __launch_bounds__(kDecThreads) decode_write_kernel(DecodeParams p)
{
    extern __shared__ __align__(16) uint32_t dec_smem[];
    uint32_t* s_fast = dec_smem;                      // [kFastWords]
    uint32_t* s_win = dec_smem + kFastWords;          // [kWinSmemWords]
    const uint32_t f = blockIdx.y, tid = threadIdx.x;
    DecodeState* stp = p.state + f;
    if (stp->status || stp->stored) return;
    const FileDesc fd = p.files[f];
    Stream sm = open_stream(p.d_files + fd.base, fd);
    const FileSpan sp = file_span(*stp, sm, fd);
    if (sp.g0 + (unsigned long long)blockIdx.x * kDecThreads > sp.g1) return;
    const unsigned long long g = sp.g0 + (unsigned long long)blockIdx.x * kDecThreads + tid;
    SubInfo in; in.nlit = 0; in.n_out = 0;
    if (g <= sp.g1) in = p.subs[fd.sub_base + (g - sp.g0)];
    // a CTA whose subsequences the link pass left dead or empty stages nothing
    if (!__syncthreads_or(in.nlit && in.n_out)) return;
    stage_fast_table(s_fast, p.fast + (size_t)f * kFastWords);
    stage_window(sm, s_win, sp.g0 + (unsigned long long)blockIdx.x * kDecThreads);
    stage_wait();
    const uint32_t* lutg = p.luts + (size_t)f * 4096;
    if (g > sp.g1) return;
    if (!in.nlit || !in.n_out) return;                                           // dead, empty or already written
    const uint32_t chans = fd.chans, bpl = fd.w * chans, h = fd.h, pitch = fd.pitch;
    uint32_t err = 0;
    const unsigned long long hi_abs = (g + 1) * kSubBits;
    if (in.start < hi_abs) {
        uint8_t* dl = p.delta + fd.delta_base;
        if (chans == 4) decode_write_range<4>(sm, s_fast, lutg, in.start, (uint32_t)(hi_abs - in.start), dl, pitch, bpl, h, in.exit /*out_pos*/, in.lits /*tail*/, &err);
        else decode_write_range<3>(sm, s_fast, lutg, in.start, (uint32_t)(hi_abs - in.start), dl, pitch, bpl, h, in.exit /*out_pos*/, in.lits /*tail*/, &err);
    }
    if (err) stp->status = 1;
}

// ------------------------------------------------------------------------------------------------
// D2': stored blocks -> delta rows (filter bytes must all be 0; "delta" then already holds final pixel bytes)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) decode_stored_kernel(DecodeParams p)
{
    const uint32_t f = blockIdx.y;
    DecodeState* st = p.state + f;
    if (st->status || !st->stored) return;
    const FileDesc fd = p.files[f];
    const uint8_t* z = p.d_files + fd.base + fd.idat_ofs + 8;
    const uint32_t avail = fd.file_size - (fd.idat_ofs + 8);
    const uint32_t bpl = fd.w * fd.chans, h = fd.h, pitch = fd.pitch;
    const unsigned long long raw = (unsigned long long)(bpl + 1) * h, nblk = (raw + 65534ull) / 65535ull;
    uint8_t* delta = p.delta + fd.delta_base;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t y = blockIdx.x * 8 + warp;
    bool bad = false;
    // block headers: every warp of block row 0 validates a strided share (fpng.cpp:2124-2146, 2195-2204)
    if (blockIdx.x == 0) {
        if (2ull + raw + 5ull * nblk + 4ull != fd.idat_len || fd.idat_len > avail) bad = true;
        else for (unsigned long long j = threadIdx.x; j < nblk; j += blockDim.x) {
            const uint8_t* b = z + 2ull + j * 65540ull;
            const unsigned long long remaining = raw - j * 65535ull;
            const uint32_t want = remaining < 65535ull ? (uint32_t)remaining : 65535u;
            const uint32_t len = b[1] | (b[2] << 8), nlen = b[3] | (b[4] << 8);
            const uint32_t fin = (j + 1 == nblk) ? 1u : 0u;
            if ((b[0] & 1u) != fin || ((b[0] >> 1) & 3u) != 0 || len != want || len != (~nlen & 0xFFFFu)) bad = true;
        }
    }
    if (y < h && !(2ull + raw + 5ull * nblk + 4ull != fd.idat_len || fd.idat_len > avail)) {
        const unsigned long long s0 = (unsigned long long)y * (bpl + 1ull);
        for (uint32_t t = lane; t <= bpl; t += 32) {
            const unsigned long long s = s0 + t;
            const uint8_t v = z[2ull + 5ull * (s / 65535ull + 1ull) + s];
            if (t == 0) { if (v != 0) bad = true; }                               // fpng.cpp:2154-2158
            else delta[(size_t)y * pitch + (t - 1)] = v;
        }
    }
    if (bad) st->status = 1;
}

// ------------------------------------------------------------------------------------------------
// V2: zlib Adler-32 of the inflated stream, read back from the delta rows (verification on only; decode.cuh, VerifyState).  It runs
// after the write and stored kernels and before unfilter_kernel, so a file whose checksum does not match gets no pixel.
// Adler-32 is linear in the byte positions: with N = h * (w*c + 1) bytes x_i at positions i = 0 .. N-1,
//     A = 1 + sum x_i,     B = N + N * sum x_i - sum i * x_i     (mod 65521),
// so any partition of the stream will do.  One warp per delta row: each lane sums the bytes of its 16-byte vectors and their
// column-weighted sum (two dp4a per word), the CTA reduces, one atomic per CTA and file adds the shares (each reduced mod 65521),
// and the file's last CTA adds the filter bytes in closed form -- 0 on the first scanline and 2 below it in compressed files, 0
// everywhere in stored files, as the write and stored kernels have checked -- and compares with the stream's last four bytes.
// ------------------------------------------------------------------------------------------------
constexpr uint32_t kAdlerRows = 8;                  // delta rows per CTA, one per warp

__global__ void __launch_bounds__(32 * kAdlerRows) decode_adler_kernel(VerifyParams p)
{
    __shared__ unsigned long long s_s1[kAdlerRows], s_s2[kAdlerRows];
    const uint32_t f = blockIdx.y, lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    if (p.state[f].status) return;                  // the same for every CTA of the file: only the last one writes it
    const FileDesc fd = p.files[f];
    const uint32_t h = fd.h, bpl = fd.w * fd.chans;
    const uint32_t nctas = (h + kAdlerRows - 1) / kAdlerRows;
    if (blockIdx.x >= nctas) return;
    const uint32_t y = blockIdx.x * kAdlerRows + warp;
    unsigned long long s1 = 0, s2 = 0;
    if (y < h) {
        const uint4* row = reinterpret_cast<const uint4*>(p.delta + fd.delta_base + (size_t)y * fd.pitch);   // 16-byte aligned
        const uint32_t nvec = (bpl + 15u) >> 4;
        uint32_t sx = 0;                            // sum of the lane's bytes
        unsigned long long sxc = 0;                 // sum of column * byte
#pragma unroll 4
        for (uint32_t v = lane; v < nvec; v += 32) {
            uint4 q = __ldg(row + v);
            const uint32_t rem = bpl - 16u * v;     // the row's pitch padding is not part of the stream
            if (rem < 16u) {
                uint32_t* w = &q.x;
#pragma unroll
                for (uint32_t k = 0; k < 4; k++) w[k] &= 4u * k >= rem ? 0u : (4u * k + 4u <= rem ? 0xFFFFFFFFu : (1u << (8u * (rem - 4u * k))) - 1u);
            }
            const uint32_t s = __dp4a(q.x, 0x01010101u, __dp4a(q.y, 0x01010101u, __dp4a(q.z, 0x01010101u, __dp4a(q.w, 0x01010101u, 0u))));
            const uint32_t t = __dp4a(q.x, 0x03020100u, __dp4a(q.y, 0x07060504u, __dp4a(q.z, 0x0B0A0908u, __dp4a(q.w, 0x0F0E0D0Cu, 0u))));
            sx += s;
            sxc += (unsigned long long)(16u * v) * s + t;
        }
        // byte x of row y is at stream position y * (bpl + 1) + 1 + x
        const unsigned long long pos0 = ((unsigned long long)y * (bpl + 1ull) + 1ull) % kAdlerMod;
        s1 = sx % kAdlerMod;
        s2 = (pos0 * s1 + sxc % kAdlerMod) % kAdlerMod;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { s1 += __shfl_xor_sync(kFullMask, s1, o); s2 += __shfl_xor_sync(kFullMask, s2, o); }
    if (lane == 0) { s_s1[warp] = s1; s_s2[warp] = s2; }
    __syncthreads();
    if (threadIdx.x != 0) return;
    s1 = 0; s2 = 0;
    for (uint32_t k = 0; k < kAdlerRows; k++) { s1 += s_s1[k]; s2 += s_s2[k]; }
    VerifyState* vs = p.vs + f;
    atomicAdd(&vs->s1, s1 % kAdlerMod);
    atomicAdd(&vs->s2, s2 % kAdlerMod);
    __threadfence();
    if (atomicAdd(&vs->adler_done, 1u) != nctas - 1) return;
    __threadfence();
    unsigned long long S1 = atomicAdd(&vs->s1, 0ull) % kAdlerMod, S2 = atomicAdd(&vs->s2, 0ull) % kAdlerMod;
    if (!p.state[f].stored && h > 1) {               // filter byte 2 at position y * (bpl + 1) of every row y >= 1
        S1 = (S1 + 2ull * (h - 1)) % kAdlerMod;
        S2 = (S2 + (bpl + 1ull) % kAdlerMod * h % kAdlerMod * (h - 1) % kAdlerMod) % kAdlerMod;   // 2 * (bpl + 1) * h (h - 1) / 2
    }
    const unsigned long long N = ((unsigned long long)h * (bpl + 1ull)) % kAdlerMod;
    const uint32_t A = (uint32_t)((1ull + S1) % kAdlerMod);
    const uint32_t B = (uint32_t)((N + N * S1 % kAdlerMod + kAdlerMod - S2) % kAdlerMod);
    const uint8_t* z = p.d_files + fd.base + fd.idat_ofs + 8;
    const uint8_t* q = z + fd.idat_len - 4;          // the write and stored kernels checked that the stream ends there
    const uint32_t want = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
    if (((B << 16) | A) != want) p.state[f].status = 102u;   // FPNGB_DECODE_ADLER_MISMATCH
}

// ------------------------------------------------------------------------------------------------
// D3: inverse Up filter (running sum down the columns) + channel conversion.  One thread per group of 4 pixels.
// ------------------------------------------------------------------------------------------------
// the 4 pixels of o[] (DST interleaved channels) as one 32-bit word per channel plane
template <int DST>
__device__ __forceinline__ void planes_of(const uint32_t (&o)[DST], uint32_t (&pl)[DST])
{
    if (DST == 4) {
        const uint32_t t01 = __byte_perm(o[0], o[1], 0x5140), t23 = __byte_perm(o[2], o[DST - 1], 0x5140);   // c0 c1 of pixels 0,1 / 2,3
        const uint32_t u01 = __byte_perm(o[0], o[1], 0x7362), u23 = __byte_perm(o[2], o[DST - 1], 0x7362);   // c2 c3
        pl[0] = __byte_perm(t01, t23, 0x5410); pl[1] = __byte_perm(t01, t23, 0x7632);
        pl[2] = __byte_perm(u01, u23, 0x5410); pl[DST - 1] = __byte_perm(u01, u23, 0x7632);
    } else {                 // o = r0 g0 b0 r1 | g1 b1 r2 g2 | b2 r3 g3 b3
        pl[0] = __byte_perm(__byte_perm(o[0], o[1], 0x0630), o[2], 0x5210);
        pl[1] = __byte_perm(__byte_perm(o[0], o[1], 0x0741), o[2], 0x6210);
        pl[2] = __byte_perm(__byte_perm(o[0], o[1], 0x0052), o[2], 0x7410);
    }
}

// Output layouts (OutStrides): interleaved rows at any pitch (PLANAR false) or one byte plane per channel (PLANAR true).  Files
// with another channel count than SRC are left to the other instantiation (the ragged call launches both).
template <int SRC, int DST, bool PLANAR>
__global__ void __launch_bounds__(128) unfilter_kernel(DecodeParams p, OutStrides os)
{
    const uint32_t f = blockIdx.y;
    const DecodeState st = p.state[f];
    if (st.status) return;
    const FileDesc& fd = p.files[f];
    if (fd.chans != SRC) return;                                                // the same for the whole CTA
    const uint32_t w = fd.w, h = fd.h, pitch = fd.pitch;
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;                   // pixel group index
    const uint32_t x0 = g * 4;
    const uint32_t amask = __ballot_sync(kFullMask, x0 < w);                     // lanes of this warp that own a group (they stay converged)
    if (x0 >= w) return;
    const uint32_t lane = threadIdx.x & 31u;
    const bool next_full = lane < 31u && x0 + 8u <= w;                           // the next lane of this warp owns a whole group
    const uint32_t npx = min(4u, w - x0);
    const uint8_t* delta = p.delta + fd.delta_base + (size_t)x0 * SRC;
    uint8_t* out = p.d_out + fd.out_base + (size_t)x0 * (PLANAR ? 1u : DST);
    const size_t out_pitch = os.row ? os.row : (size_t)w * DST, cs = os.chan;
    const bool full = npx == 4;
    const bool out_aligned = (((uintptr_t)out | out_pitch) & 3) == 0;
    uint32_t acc[SRC];
#pragma unroll
    for (int i = 0; i < SRC; i++) acc[i] = 0;
    const bool summing = !st.stored;
    constexpr int kRowsAhead = 8;                  // independent loads in flight per thread (8 rows x 12-16 bytes: enough bytes in flight at 256 files)
    for (uint32_t y0 = 0; y0 < h; y0 += kRowsAhead) {
        uint32_t dd[kRowsAhead][SRC];
        load_delta_rows<SRC>(delta, pitch, y0, h, full, npx, dd);
#pragma unroll
        for (int j = 0; j < kRowsAhead; j++) {
            const uint32_t y = y0 + j;
            if (y >= h) break;
            uint32_t o[DST];
            unfilter_row<SRC, DST>(acc, dd[j], summing, o);
            uint8_t* orow = out + (size_t)y * out_pitch;
            if (PLANAR) {
                // one word per plane when every plane row is 4-byte aligned (x0 % 4 == 0), else bytes
                uint32_t pl[DST];
                planes_of<DST>(o, pl);
                if (full && ((((uintptr_t)orow) | cs) & 3u) == 0u) {
#pragma unroll
                    for (int c = 0; c < DST; c++) *reinterpret_cast<uint32_t*>(orow + c * cs) = pl[c];
                } else {
#pragma unroll
                    for (int c = 0; c < DST; c++) for (uint32_t b = 0; b < npx; b++) orow[c * cs + b] = (uint8_t)(pl[c] >> (8u * b));
                }
                continue;
            }
            // output scanlines of any width (w * DST need not be a multiple of 4: 687 x 3 = 2061): the misalignment is the same for every
            // group of a scanline (groups are 4 * DST bytes apart), so the aligned words a thread's bytes straddle are assembled with
            // one funnel shift each, the word shared with the previous group from that lane's last word (shuffle); only the two ends
            // of a warp's stretch go out as single bytes
            const uint32_t prev_last = __shfl_up_sync(amask, o[DST - 1], 1);
            const uint32_t mis = (uint32_t)((uintptr_t)orow & 3u);
            if (full && (out_aligned || mis == 0u)) {
#pragma unroll
                for (int i = 0; i < DST; i++) *reinterpret_cast<uint32_t*>(orow + 4 * i) = o[i];
            } else if (full) {
                const uint32_t sh = 8u * (4u - mis);
                uint8_t* ab = orow - mis;                                        // 4-byte aligned
                if (lane > 0u) *reinterpret_cast<uint32_t*>(ab) = __funnelshift_r(prev_last, o[0], sh);
                else for (uint32_t b = 0; b < 4u - mis; b++) orow[b] = (uint8_t)(o[0] >> (8u * b));
#pragma unroll
                for (int i = 1; i < DST; i++) *reinterpret_cast<uint32_t*>(ab + 4 * i) = __funnelshift_r(o[i - 1], o[i], sh);
                if (!next_full) for (uint32_t b = 0; b < mis; b++) orow[4u * DST - mis + b] = (uint8_t)(o[DST - 1] >> (8u * (4u - mis + b)));
            } else {
#pragma unroll
                for (int i = 0; i < DST; i++) for (int b = 0; b < 4; b++) if ((uint32_t)(4 * i + b) < npx * DST) orow[4 * i + b] = (uint8_t)(o[i] >> (8 * b));
            }
        }
    }
}


__global__ void decode_status_kernel(DecodeParams p, uint32_t n)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < n) {
        const uint32_t pre = p.files[f].pre_status;
        p.d_status[f] = pre ? pre : p.state[f].status;   // 0, 1 (FPNG_DECODE_NOT_FPNG), or a verify kernel's 4 / 102
    }
}

// Optional per-kernel timing of the decode pipeline (bench.py): events recorded between the launches of the most recent
// call while profiling is on; fpngb_decode_profile_read() returns the device times of prepare, scan, link, write, stored,
// unfilter (ms), and for a verified call also the IDAT CRC (slot 6) and Adler-32 (slot 7) kernels.  Events 0..6 bound the six
// slots; a verified call also records event 7 after the CRC kernel (scan then starts there) and event 8 after the Adler kernel
// (unfilter then starts there).  The resized call records event 10 right before its resize kernel (behind the any-PNG kernels
// when it has them) and event 9 after it: slot 8, with slots 6 and 7 0 when the call is not verified.
static bool g_dec_profile = false;
static cudaEvent_t g_dec_ev[11];
static bool g_dec_ev_ready = false, g_dec_ev_valid = false, g_dec_ev_verify = false, g_dec_ev_resize = false;
void decode_profile_enable(bool on)
{
    g_dec_profile = on;
    if (on && !g_dec_ev_ready) { for (int i = 0; i < 11; i++) cudaEventCreate(&g_dec_ev[i]); g_dec_ev_ready = true; }
}
int decode_profile_read(float* ms, int n)
{
    if (!g_dec_ev_valid) return 0;
    cudaEventSynchronize(g_dec_ev[g_dec_ev_resize ? 9 : 6]);
    int from[9] = {0, 1, 2, 3, 4, 5, 1, 5, 10}, to[9] = {1, 2, 3, 4, 5, 6, 7, 8, 9};
    if (g_dec_ev_verify) { from[1] = 7; from[5] = 8; }
    const int slots = g_dec_ev_resize ? 9 : g_dec_ev_verify ? 8 : 6;
    for (int i = 0; i < n && i < slots; i++) {
        ms[i] = 0.f;
        if (i < 6 || i == 8 || g_dec_ev_verify) cudaEventElapsedTime(&ms[i], g_dec_ev[from[i]], g_dec_ev[to[i]]);
    }
    return 1;
}
#define DEC_MARK(i) do { if (g_dec_profile && g_dec_ev_ready) cudaEventRecord(g_dec_ev[i], s); } while (0)
void decode_profile_mark_resize(cudaStream_t s, bool done)
{
    DEC_MARK(done ? 9 : 10);
    if (done && g_dec_profile && g_dec_ev_ready) g_dec_ev_resize = true;
}

// Speculative lead-in of decode_scan_kernel (fpngb_debug_decode_preroll).  The link pass makes the result independent of it; tests set
// it below the default to force wrong guesses.  At most kPreRoll: the scan kernel's stream window starts kWinLead words before its
// first subsequence.
static_assert(kPreRoll <= kWinLead * 32, "the pre-roll stays inside the scan kernel's stream window");
static uint32_t g_dec_pre_roll = kPreRoll;
bool decode_set_pre_roll(uint32_t bits)
{
    if (bits > kPreRoll) return false;
    g_dec_pre_roll = bits;
    return true;
}

void launch_decode(const DecodeParams& params, const OutStrides& os, uint32_t n, uint32_t desired, cudaStream_t s, VerifyState* verify,
                   size_t max_file_bytes, const TypedOut* typed)
{
    DecodeParams p = params;
    p.pre_roll = g_dec_pre_roll;
    const VerifyParams vp{p.d_files, p.files, p.state, p.delta, verify};
    if (verify) cudaMemsetAsync(verify, 0, (size_t)n * sizeof(VerifyState), s);
    DEC_MARK(0);
    decode_prepare_kernel<<<n, 32, 0, s>>>(p);
    DEC_MARK(1);
    if (verify) {                                   // after prepare (which resets the state), before anything decodes the stream
        launch_idat_crc_verify(vp, n, max_file_bytes, s);
        DEC_MARK(7);
    }
    const uint32_t sub_blocks = (p.max_subs + kDecThreads - 1) / kDecThreads;
    dim3 gsub(sub_blocks, n);
    constexpr size_t kDecSmem = (kFastWords + kWinSmemWords) * 4;
    FPNGB_SET_SMEM(decode_scan_kernel, kDecSmem);
    FPNGB_SET_SMEM(decode_write_kernel, kDecSmem);
    decode_scan_kernel<<<gsub, kDecThreads, kDecSmem, s>>>(p);
    DEC_MARK(2);
    decode_link_kernel<<<n, kLinkThreads, 0, s>>>(p);
    DEC_MARK(3);
    decode_write_kernel<<<gsub, kDecThreads, kDecSmem, s>>>(p);
    DEC_MARK(4);
    dim3 gs((p.max_h + 7) / 8, n);
    decode_stored_kernel<<<gs, 256, 0, s>>>(p);
    DEC_MARK(5);
    if (verify) {                                   // every delta row is final; no pixel is written yet
        decode_adler_kernel<<<dim3((p.max_h + kAdlerRows - 1) / kAdlerRows, n), 32 * kAdlerRows, 0, s>>>(vp);
        DEC_MARK(8);
    }
    const uint32_t groups = (p.max_w + 3) / 4;
    dim3 gu((groups + 127) / 128, n);
    const bool planar = os.pixel == 1;
    if (typed) launch_unfilter_typed(p, os, *typed, desired, gu, s);
    // one instantiation per channel count in the call (a mixed call launches both; each skips the other's files)
    for (uint32_t src = 3; src <= 4 && !typed; src++) {
        if (p.chans && p.chans != src) continue;
        if (src == 3 && desired == 3) { if (planar) unfilter_kernel<3, 3, true><<<gu, 128, 0, s>>>(p, os); else unfilter_kernel<3, 3, false><<<gu, 128, 0, s>>>(p, os); }
        else if (src == 3) { if (planar) unfilter_kernel<3, 4, true><<<gu, 128, 0, s>>>(p, os); else unfilter_kernel<3, 4, false><<<gu, 128, 0, s>>>(p, os); }
        else if (desired == 3) { if (planar) unfilter_kernel<4, 3, true><<<gu, 128, 0, s>>>(p, os); else unfilter_kernel<4, 3, false><<<gu, 128, 0, s>>>(p, os); }
        else { if (planar) unfilter_kernel<4, 4, true><<<gu, 128, 0, s>>>(p, os); else unfilter_kernel<4, 4, false><<<gu, 128, 0, s>>>(p, os); }
    }
    decode_status_kernel<<<(n + 127) / 128, 128, 0, s>>>(p, n);
    DEC_MARK(6);
    if (g_dec_profile && g_dec_ev_ready) { g_dec_ev_valid = true; g_dec_ev_verify = verify != nullptr; g_dec_ev_resize = false; }
}

}  // namespace fpngb
