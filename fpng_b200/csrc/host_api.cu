// fpng_b200/csrc/host_api.cu -- host runtime + C ABI (include/fpng_b200.h) of the H100 (sm_90a) fpng hot path.
//
// The host side owns: the CUDA context/stream, the static (1-pass) code books derived from the format's
// pre-serialised block headers, a grow-only device workspace, the 58-byte container header template, and the
// H2D/D2H plumbing for host-buffer callers.  All pixel/bit work runs in the kernels of encode_kernels.cu,
// checksum_kernels.cu, huffman_kernels.cu and decode_kernels.cu.  There is no CPU fallback: without a CUDA
// device every entry point fails with FPNGB_ERR_NO_DEVICE.
#include "../../include/fpng_b200.h"
#include "kernels.cuh"
#include "crc_math.cuh"
#include "layout.h"
#include "row_walk.cuh"
#include "static_tables.h"
#include "runtime.h"

#include <algorithm>
#include <atomic>
#include <mutex>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

namespace fpngb {

static std::atomic<uint64_t> g_launches{0};

static bool g_pack_crc = true;                  // fpngb_debug_pack_crc(): the 16-pixel pack kernel computes scanline CRCs (no CRC pass over the file)
static bool g_fused = false;                    // fpngb_debug_use_fused(1): the single-pass encoder instead of the two-kernel encoder
static bool g_crc_overlap = false;              // fpngb_debug_crc_overlap(1): chunked batches with the CRC kernel on a side stream (off by default: measured slower than the serial order)
void count_launch(uint64_t n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

// ---------------------------------------------------------------------------------------------------------
// Static code books: parse "HLIT HDIST HCLEN, code-length code, RLE'd code sizes" exactly as an inflater does
// (RFC 1951 3.2.7; the reference's own reader is fpng.cpp:1954-2076) and assign canonical codes (fpng.cpp:701-708).
// ---------------------------------------------------------------------------------------------------------
struct BitReader {
    const uint8_t* p; uint32_t nbits; uint32_t pos = 0; bool bad = false;
    uint32_t get(int n)
    {
        uint32_t v = 0;
        for (int i = 0; i < n; i++) {
            if (pos >= nbits) { bad = true; return 0; }
            v |= (uint32_t)((p[pos >> 3] >> (pos & 7)) & 1) << i;
            pos++;
        }
        return v;
    }
};

static uint32_t reverse_bits(uint32_t v, int n) { uint32_t r = 0; for (int i = 0; i < n; i++) { r = (r << 1) | ((v >> i) & 1); } return r; }

static void canonical_codes(const uint8_t* sizes, int n, uint16_t* codes)
{
    uint32_t count[16] = {0}, next[16] = {0};
    for (int i = 0; i < n; i++) count[sizes[i]]++;
    count[0] = 0;
    for (int l = 1; l < 16; l++) next[l] = (next[l - 1] + count[l - 1]) << 1;
    for (int i = 0; i < n; i++) codes[i] = sizes[i] ? (uint16_t)reverse_bits(next[sizes[i]]++, sizes[i]) : 0;
}

static bool read_code_sizes(BitReader& br, uint8_t* lit_sizes /*288*/, uint8_t* dist_sizes /*32*/)
{
    static const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    const uint32_t nlit = br.get(5) + 257, ndist = br.get(5) + 1, nclen = br.get(4) + 4;
    uint8_t cl[19] = {0};
    for (uint32_t i = 0; i < nclen; i++) cl[order[i]] = (uint8_t)br.get(3);
    uint16_t clcodes[19];
    canonical_codes(cl, 19, clcodes);
    uint8_t all[288 + 32] = {0};
    uint32_t cur = 0;
    while (cur < nlit + ndist && !br.bad) {
        // decode one code-length symbol bit by bit (tiny table: linear search is fine at init time)
        uint32_t code = 0; int len = 0, sym = -1;
        while (sym < 0 && len < 8) {
            code |= br.get(1) << len; len++;
            for (int s = 0; s < 19; s++) if (cl[s] == len && clcodes[s] == code) { sym = s; break; }
        }
        if (sym < 0) return false;
        if (sym < 16) { all[cur++] = (uint8_t)sym; continue; }
        uint32_t rep, val = 0;
        if (sym == 16) { rep = br.get(2) + 3; if (!cur) return false; val = all[cur - 1]; }
        else if (sym == 17) rep = br.get(3) + 3;
        else rep = br.get(7) + 11;
        if (cur + rep > nlit + ndist) return false;
        while (rep--) all[cur++] = (uint8_t)val;
    }
    if (br.bad) return false;
    memset(lit_sizes, 0, 288); memset(dist_sizes, 0, 32);
    memcpy(lit_sizes, all, nlit); memcpy(dist_sizes, all + nlit, ndist);
    return true;
}

// Fill the kernel-facing tables of a code book from lit/len code sizes + codes.
void finish_codebook(CodeBook& cb, const uint8_t* sizes, const uint16_t* codes, uint32_t chans)
{
    for (int v = 0; v < 256; v++) { cb.lit[v] = codes[v] | ((uint32_t)sizes[v] << 16); cb.lit_size[v] = sizes[v]; }
    memset(cb.match, 0, sizeof cb.match); memset(cb.match_bits, 0, sizeof cb.match_bits);
    const uint32_t M = max_match_pixels(chans);
    for (uint32_t n = 1; n <= M; n++) {
        uint32_t sym, xb, xv;
        deflate_len_code(n * chans, sym, xb, xv);
        const uint32_t s = sizes[sym], total = s + xb + 1;          // +1: the 1-bit distance code, always 0 (fpng.cpp:1135)
        cb.match[n] = (codes[sym] | (xv << s)) | (total << 24);
        cb.match_bits[n] = (uint8_t)total;
    }
    cb.eob = codes[256] | ((uint32_t)sizes[256] << 16);
    memcpy(cb.sym_size, sizes, 288);
}

static bool build_static_book(CodeBook& cb, const uint8_t* hdr, uint32_t nbytes, uint32_t tail, uint32_t tail_bits, uint32_t chans)
{
    memset(&cb, 0, sizeof cb);
    memcpy(cb.hdr, hdr, nbytes);
    cb.hdr[nbytes] = (uint8_t)tail;
    cb.hdr_bits = nbytes * 8 + tail_bits;
    BitReader br{cb.hdr, cb.hdr_bits};
    br.pos = 16;
    if (br.get(1) != 1 || br.get(2) != 2) return false;
    uint8_t lit_sizes[288], dist_sizes[32];
    if (!read_code_sizes(br, lit_sizes, dist_sizes) || br.pos != cb.hdr_bits) return false;
    // fpng decoders (fpng.cpp:2007, 2058-2074) accept literal/length code sizes up to 12 only, and the pack kernels
    // hard-code the distance code as the single bit 0: exactly the table the trainer emits (fpng.cpp:1096-1098) --
    // 1-bit codes at distance symbols chans-1 (code 0) and optionally chans (code 1), nothing else.
    for (int v = 0; v < 288; v++) if (lit_sizes[v] > 12) return false;
    for (uint32_t d = 0; d < 32; d++) {
        const bool allowed = d == chans - 1 || d == chans;
        if (dist_sizes[d] != 0 && !(allowed && dist_sizes[d] == 1)) return false;
    }
    if (dist_sizes[chans - 1] != 1) return false;
    uint16_t codes[288];
    canonical_codes(lit_sizes, 288, codes);
    const uint32_t M = max_match_pixels(chans);
    for (uint32_t n = 1; n <= M; n++) { uint32_t s, xb, xv; deflate_len_code(n * chans, s, xb, xv); if (!lit_sizes[s]) return false; }
    for (int v = 0; v <= 256; v++) if (!lit_sizes[v]) return false;
    finish_codebook(cb, lit_sizes, codes, chans);
    // can "size(len sym 258) + 1 > sum of four literal sizes" (fpng.cpp:1520-1528) ever hold under this table?
    uint32_t min_lit = 255;
    for (int v = 0; v < 256; v++) min_lit = lit_sizes[v] < min_lit ? lit_sizes[v] : min_lit;
    cb.lit1_rule = (chans == 4 && cb.match_bits[1] > 4u * min_lit) ? 1 : 0;
    return true;
}

// ---------------------------------------------------------------------------------------------------------
// Context
// ---------------------------------------------------------------------------------------------------------
static Context g_ctx;
static std::mutex g_init_mu;
Context& context() { return g_ctx; }

// Optional per-kernel timing with CUDA events on the launching stream (bench.py's roofline numbers).
// kProfConvert: the conversion pre-pass (convert_pixels_kernel), which runs before the first slot and has its own start event.
// kProfReduce: the colour-type analysis of FPNGB_ENCODE_REDUCE (analysis and palette finalise), before the conversion, own start event.
// kProfMatch: the LZ77 match kernel, between the filter pass (kProfHist) and the Huffman build (kProfHuff), which then starts at its end.
enum ProfSlot { kProfHist = 0, kProfHuff, kProfScan, kProfOffsets, kProfFused, kProfFinish, kProfPack, kProfAdler, kProfCrc, kProfConvert,
                kProfReduce, kProfMatch, kProfSlots };
struct ProfSet {
    cudaEvent_t ev[kProfSlots + 1]; cudaEvent_t crc_start, conv_start, red_start; bool used[kProfSlots]; bool crc_side; uint64_t call;
};
static uint64_t g_prof_call = 0;                // encode calls seen while profiling (a chunked call owns several ProfSets)
static bool g_profile = false;
static std::vector<ProfSet*> g_prof_sets;      // one per encode call since the last read
static std::vector<ProfSet*> g_prof_free;
static ProfSet* g_prof_conv = nullptr;         // a set whose conversion slot is recorded; the next prof_begin takes it over

static ProfSet* prof_alloc()
{
    ProfSet* ps;
    if (!g_prof_free.empty()) { ps = g_prof_free.back(); g_prof_free.pop_back(); }
    else {
        ps = new ProfSet();
        for (int i = 0; i <= kProfSlots; i++) if (cudaEventCreate(&ps->ev[i]) != cudaSuccess) { delete ps; return nullptr; }
        if (cudaEventCreate(&ps->crc_start) != cudaSuccess || cudaEventCreate(&ps->conv_start) != cudaSuccess ||
            cudaEventCreate(&ps->red_start) != cudaSuccess) { delete ps; return nullptr; }
    }
    ps->crc_side = false;
    for (int i = 0; i < kProfSlots; i++) ps->used[i] = false;
    return ps;
}

static ProfSet* prof_begin(cudaStream_t s)
{
    if (!g_profile) return nullptr;
    ProfSet* ps = g_prof_conv ? g_prof_conv : prof_alloc();
    g_prof_conv = nullptr;
    if (!ps) return nullptr;
    ps->call = g_prof_call;
    cudaEventRecord(ps->ev[0], s);
    g_prof_sets.push_back(ps);
    return ps;
}

// a conversion slot no encode took over (the call failed after the pre-pass) is dropped
static void prof_drop_conv()
{
    if (g_prof_conv) { g_prof_free.push_back(g_prof_conv); g_prof_conv = nullptr; }
}
// records the end of slot `slot`; slots must be closed in increasing order, skipped slots stay unused
static void prof_mark(ProfSet* ps, int slot, cudaStream_t s)
{
    if (!ps) return;
    cudaEventRecord(ps->ev[slot + 1], s);
    ps->used[slot] = true;
}

// The conversion descriptor of n images of one shape in byte layout L whose tight rows of sample_bytes-byte samples go to byte dst
// of the conversion buffer, converted by the CTAs from cta_start on.
static ConvDesc conv_desc(const uint8_t* src, const Layout& L, uint32_t n, uint32_t w, uint32_t h, uint32_t chans, uint64_t dst,
                          uint64_t cta_start, uint32_t sample_bytes = 1)
{
    return ConvDesc{src, L.image, L.row, L.chan, dst, cta_start, n, w, h, chans, convert_ctas_per_image(w, h), L.planar ? 1u : 0u,
                    sample_bytes};
}

// One launch of the conversion pre-pass over the count descriptors hd (ascending cta_start; for count > 1 also uploaded to d_desc)
// into tight rows at dst, the uint8 copy for f.dtype 0; png: the PNG call's instantiations (1 to 4 channels, 8- or 16-bit samples).
// Profiled in slot kProfConvert of the encode that follows it on the stream.
static void convert_enqueue(const ConvDesc* hd, uint32_t count, const ConvDesc* d_desc, const PixelFormat& f, uint8_t* dst, cudaStream_t s,
                            bool png = false)
{
    ConvertParams cp{};
    cp.one = hd[0]; cp.desc = d_desc; cp.count = count; cp.dst = dst;
    cp.total_ctas = hd[count - 1].cta_start + (unsigned long long)hd[count - 1].n * hd[count - 1].ctas_per_image;
    memcpy(cp.scale, f.scale, sizeof cp.scale); memcpy(cp.bias, f.bias, sizeof cp.bias);
    uint32_t planar = 0;
    for (uint32_t i = 0; i < count; i++) planar += hd[i].planar;
    prof_drop_conv();
    ProfSet* ps = g_profile ? prof_alloc() : nullptr;
    if (ps) cudaEventRecord(ps->conv_start, s);
    launch_convert_pixels(cp, f.dtype, planar == 0 ? kConvInterleaved : planar == count ? kConvPlanar : kConvAny, png, s);
    count_launch(1);
    if (ps) { prof_mark(ps, kProfConvert, s); g_prof_conv = ps; }
}

struct Workspace {
    uint32_t* row_bits; uint2* row_adler; unsigned long long* row_ofs; ImageState* st; uint32_t* hist; CodeBook* books;
    uint2* lane_ofs; uint32_t lane_ofs_pitch;
    void* fused_desc;
    uint32_t* row_crc;
};


static int carve_workspace(Context& c, uint32_t n, uint32_t h, uint32_t width, bool two_pass, Workspace& w, bool fused = false)
{
    const size_t rows = (size_t)n * h;
    const uint32_t lane_pitch = ((width + 511u) / 512u) * 32u;       // one uint2 per 16-pixel group, whole warp steps
    size_t o = 0;
    const size_t o_bits = o; o = align_up(o + rows * 4, 256);
    const size_t o_adl = o; o = align_up(o + rows * 8, 256);
    const size_t o_ofs = o; o = align_up(o + rows * 8, 256);
    const size_t o_st = o; o = align_up(o + (size_t)n * sizeof(ImageState), 256);
    const size_t o_hist = o; o = align_up(o + (two_pass ? (size_t)n * 288 * 4 : 0), 256);
    const size_t o_books = o; o = align_up(o + (two_pass ? (size_t)n * sizeof(CodeBook) : 0), 256);
    const size_t o_lane = o; o = align_up(o + (fused ? 0 : rows * lane_pitch * 8), 256);
    const size_t o_desc = o; o = align_up(o + (fused ? fused_desc_bytes(n, width, h) : 0), 256);
    const size_t o_rcrc = o; o = align_up(o + (fused ? 0 : rows * 4), 256);
    int rc = c.ws.reserve(o);
    if (rc) return rc;
    uint8_t* b = (uint8_t*)c.ws.p;
    w.row_crc = (uint32_t*)(b + o_rcrc);
    w.row_bits = (uint32_t*)(b + o_bits); w.row_adler = (uint2*)(b + o_adl); w.row_ofs = (unsigned long long*)(b + o_ofs);
    w.st = (ImageState*)(b + o_st); w.hist = (uint32_t*)(b + o_hist); w.books = (CodeBook*)(b + o_books);
    w.lane_ofs = (uint2*)(b + o_lane); w.lane_ofs_pitch = lane_pitch;
    w.fused_desc = b + o_desc;
    return 0;
}

static bool valid_dims(uint32_t w, uint32_t h, uint32_t chans)
{
    // fpng.cpp:1670-1680; additionally the filtered stream must be addressable with 32 bits like the reference's
    // own uint32 offsets (SURVEY Q7).
    if (w < 1 || h < 1 || (uint64_t)w * h > 0xFFFFFFFFull || w > (1u << 24) || h > (1u << 24)) return false;
    if (chans != 3 && chans != 4) return false;
    if (((uint64_t)w * chans + 1) * h + 1024 > 0xFFFFFFFFull) return false;
    return true;
}

static void make_png_header(uint8_t* hdr, uint32_t w, uint32_t h, uint32_t chans)
{
    // fpng.cpp:1770-1783 (Appendix A of SURVEY.md).  Width/height are written as full big-endian 32-bit values
    // (the reference only writes the low 16 bits, Q1: identical for every dimension < 65536).
    static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};
    static const uint8_t fdec[17] = {0, 0, 0, 5, 'f', 'd', 'E', 'C', 82, 36, 147, 227, 0, 0xE5, 0xAB, 0x62, 0x99};
    memset(hdr, 0, kPngHeaderSize);
    memcpy(hdr, sig, 8);
    hdr[11] = 13; memcpy(hdr + 12, "IHDR", 4);
    for (int i = 0; i < 4; i++) { hdr[16 + i] = (uint8_t)(w >> (24 - 8 * i)); hdr[20 + i] = (uint8_t)(h >> (24 - 8 * i)); }
    hdr[24] = 8; hdr[25] = chans == 3 ? 2 : 6;
    const uint32_t c = host_crc32(hdr + 12, 17, 0);
    for (int i = 0; i < 4; i++) hdr[29 + i] = (uint8_t)(c >> (24 - 8 * i));
    memcpy(hdr + 33, fdec, 17);
    memcpy(hdr + 54, "IDAT", 4);            // bytes 50..53 (IDAT length) are patched per image on the device
}

// Enqueue the whole encode pipeline for a device-resident batch.  Caller holds ctx.mu.
//
// Two encoders share this entry:
//  * the two-kernel encoder (scan -> offsets -> pack -> adler -> crc), the default.  Optionally (fpngb_debug_crc_overlap) large
//    batches are cut into chunks and the CRC kernel of chunk k runs on a side stream underneath the scan and pack kernels of
//    chunk k + 1 -- measured slower than the serial order (the kernels slow each other down more than the overlap gains),
//    so it is off by default;
//  * the single-pass encoder (encode_fused.cu), selected with fpngb_debug_use_fused(1): reads the pixels once
//    and writes the file once, byte-identical output, measured slower than the two-kernel path because it is bound by
//    instruction issue, not by HBM.
//
// The input is n images of format f at src in byte layout L (layout.h; a uint8 row pitch fits in 32 bits).  The scan and pack
// kernels read every uint8 layout in place.  The conversion pre-pass (convert_pixels_kernel) first writes tight uint8 rows into
// c.conv for a float input, and for a uint8 input that is not tight interleaved but bound for the single-pass encoder, which reads
// tight interleaved rows only.  Rows already in c.conv are tight uint8, so they are never converted again.
static int encode_batch_locked(Context& c, const uint8_t* src, const Layout& L, const PixelFormat& f, uint32_t n, uint32_t w, uint32_t h,
                               uint32_t chans, uint32_t flags, uint8_t* d_out, size_t out_stride, uint32_t* d_sizes, cudaStream_t s)
{
    const bool two_pass = (flags & FPNGB_ENCODE_SLOWER) && !(flags & FPNGB_FORCE_UNCOMPRESSED);
    // RGBA 1-pass under a table where a one-pixel match can lose against four literals (fpng.cpp:1520-1528; never with the shipped
    // table): the scan and pack kernels' LIT1 instantiations; the single-pass encoder does not implement the rule
    const uint32_t lit1_rule = (!two_pass && chans == 4 && c.h_static_books[1].lit1_rule) ? 1u : 0u;
    const bool fused = g_fused && !lit1_rule && !(flags & FPNGB_FORCE_UNCOMPRESSED) && fused_eligible(src, L.image, w, h, chans, n);
    const bool convert = f.dtype != 0 || (fused && (L.planar || L.row != (uint64_t)w * chans));
    const size_t image_bytes = (size_t)w * h * chans;
    Workspace ws;
    int rc = carve_workspace(c, n, h, w, two_pass, ws, fused);
    if (rc) return rc;
    if (convert) { rc = c.conv.reserve((size_t)n * image_bytes); if (rc) return rc; }
    rc = c.ws_acquire(s);
    if (rc) return rc;
    const uint8_t* d_pixels = convert ? (const uint8_t*)c.conv.p : src;
    const size_t image_stride = convert ? image_bytes : L.image, chan_stride = convert || !L.planar ? 0 : L.chan;
    const uint32_t row_pitch = convert ? w * chans : (uint32_t)L.row;
    const CodeBook* books0 = two_pass ? ws.books : c.d_static_books + (chans == 4 ? 1 : 0);
    const uint32_t book_stride = two_pass ? 1u : 0u;
    const uint32_t merge_first_unit = (!two_pass && chans == 3) ? 1u : 0u;
    uint8_t png_header[kPngHeaderSize];
    make_png_header(png_header, w, h, chans);
    if (g_profile) g_prof_call++;

    // chunks: the CRC of one chunk overlaps the scan/pack of the next.  Small batches (and the single-pass encoder) run as one chunk.
    const uint32_t nchunks = (!fused && g_crc_overlap && n >= 16) ? 4u : 1u;
    if (nchunks > 1) {
        if (!c.side) FPNGB_CUDA_OK(cudaStreamCreateWithFlags(&c.side, cudaStreamNonBlocking));
        for (int i = 0; i < 5; i++) if (!c.side_ev[i]) FPNGB_CUDA_OK(cudaEventCreateWithFlags(&c.side_ev[i], cudaEventDisableTiming));
    }
    // nothing can fail between the pre-pass and the first chunk's prof_begin, which takes over its profile slot
    if (convert) {
        const ConvDesc d = conv_desc(src, L, n, w, h, chans, 0, 0);
        convert_enqueue(&d, 1, nullptr, f, (uint8_t*)c.conv.p, s);
    }
    for (uint32_t k = 0; k < nchunks; k++) {
        const uint32_t i0 = (uint32_t)((uint64_t)n * k / nchunks), i1 = (uint32_t)((uint64_t)n * (k + 1) / nchunks), cnt = i1 - i0;
        if (!cnt) continue;
        const uint8_t* px = d_pixels + (size_t)i0 * image_stride;
        uint8_t* out = d_out + (size_t)i0 * out_stride;
        const CodeBook* books = books0 + (size_t)i0 * book_stride;
        const size_t r0 = (size_t)i0 * h;

        ScanParams sp{};
        sp.pixels = px; sp.image_stride = image_stride; sp.row_pitch = row_pitch; sp.chan_stride = chan_stride; sp.w = w; sp.h = h;
        sp.books = books; sp.book_stride = book_stride;
        sp.row_bits = ws.row_bits + r0; sp.row_adler = ws.row_adler + r0; sp.st = ws.st + i0; sp.hist = ws.hist + (size_t)i0 * 288;
        sp.merge_first_unit = merge_first_unit;
        sp.lane_ofs = ws.lane_ofs + r0 * ws.lane_ofs_pitch; sp.lane_ofs_pitch = ws.lane_ofs_pitch;
        sp.lit1_rule = lit1_rule;

        ProfSet* ps = prof_begin(s);
        if (two_pass) {
            FPNGB_CUDA_OK(cudaMemsetAsync(sp.hist, 0, (size_t)cnt * 288 * 4, s));
            launch_hist16(sp, cnt, chans, s);
            prof_mark(ps, kProfHist, s);
            HuffParams hp{sp.hist, ws.books + i0, chans, 0u};
            launch_huffman_build(hp, cnt, s);
            prof_mark(ps, kProfHuff, s);
            count_launch(2);
        }
        PackParams pp{};
        pp.pixels = px; pp.image_stride = image_stride; pp.row_pitch = row_pitch; pp.chan_stride = chan_stride; pp.w = w; pp.h = h; pp.books = books; pp.book_stride = book_stride;
        pp.row_ofs = ws.row_ofs + r0; pp.row_bits = sp.row_bits; pp.lane_ofs = sp.lane_ofs; pp.lane_ofs_pitch = ws.lane_ofs_pitch;
        pp.row_adler = sp.row_adler; pp.st = sp.st; pp.out = out; pp.out_stride = out_stride;
        pp.lit1_rule = lit1_rule;
        // the 16-pixel pack kernel computes each scanline's CRC while its code words are staged; the file is not read back
        const bool pack_crc = !fused && g_pack_crc;
        if (pack_crc) { pp.row_crc = ws.row_crc + r0; pp.crc_f128b = c.crc_f128b; pp.crc_lane_mul = c.crc_lane_mul; }
        if (fused) {
            cudaEvent_t mid = ps ? ps->ev[kProfFused + 1] : nullptr;
            rc = launch_encode_fused(px, image_stride, cnt, w, h, chans, flags, books, book_stride, sp.row_adler, sp.st, ws.fused_desc,
                                     out, out_stride, d_sizes + i0, png_header, merge_first_unit, s, mid);
            if (rc) return rc;
            if (ps) ps->used[kProfFused] = true;
            prof_mark(ps, kProfFinish, s);
            pp.stored_only = 1u;
            launch_pack16(pp, cnt, chans, s);                                   // stored-block images only (fpng.cpp:1728-1758)
            prof_mark(ps, kProfPack, s);
            count_launch(3);
        } else {
            launch_scan16(sp, cnt, chans, s);
            prof_mark(ps, kProfScan, s);
            OffsetsParams op{};
            op.row_bits = sp.row_bits; op.row_ofs = ws.row_ofs + r0; op.books = books; op.book_stride = book_stride; op.st = sp.st;
            op.out = out; op.out_stride = out_stride; op.sizes = d_sizes + i0; op.w = w; op.h = h; op.chans = chans; op.flags = flags;
            memcpy(op.png_header, png_header, kPngHeaderSize);
            launch_offsets(op, cnt, s);
            prof_mark(ps, kProfOffsets, s);
            launch_pack16(pp, cnt, chans, s);
            prof_mark(ps, kProfPack, s);
            count_launch(3);
        }
        AdlerParams ap{sp.row_adler, sp.st, out, out_stride, w, h, chans};
        launch_adler_finalize(ap, cnt, s);
        prof_mark(ps, kProfAdler, s);

        CrcParams cp{};
        cp.out = out; cp.out_stride = out_stride; cp.st = sp.st;
        cudaStream_t cs = s;
        if (nchunks > 1) {                                                    // this chunk's CRC goes to the side stream
            FPNGB_CUDA_OK(cudaEventRecord(c.side_ev[k], s));
            FPNGB_CUDA_OK(cudaStreamWaitEvent(c.side, c.side_ev[k], 0));
            cs = c.side;
            if (ps) { cudaEventRecord(ps->crc_start, cs); ps->crc_side = true; }
        }
        if (fused) {
            launch_fused_crc(ws.fused_desc, cnt, w, h, books, book_stride, sp.st, out, out_stride, cs);   // combine the in-kernel partials
            cp.stored_only = 1u;                                              // the file-reading CRC kernel is only needed for stored-block images
            count_launch(1);
        }
        if (pack_crc) {
            RowCrcParams rp{pp.row_crc, pp.row_ofs, pp.row_bits, books, book_stride, sp.st, out, out_stride, h};
            launch_row_crc_combine(rp, cnt, cs);
            cp.stored_only = 1u;
            count_launch(1);
        }
        launch_crc_stream(cp, cnt, max_encoded_size(w, h, chans), cs);
        prof_mark(ps, kProfCrc, cs);
        count_launch(2);
    }
    if (nchunks > 1) {                                                        // join: the caller's stream continues after the last CRC
        FPNGB_CUDA_OK(cudaEventRecord(c.side_ev[4], c.side));
        FPNGB_CUDA_OK(cudaStreamWaitEvent(s, c.side_ev[4], 0));
    }
    FPNGB_CUDA_OK(cudaGetLastError());
    return c.ws_release(s);
}

// ---------------------------------------------------------------------------------------------------------
// Ragged encode: images of any shape and layout in one call (fpngb_encode_ragged_device).
// ---------------------------------------------------------------------------------------------------------
// One image as the host sees it after the call-level checks.
struct RaggedImage {
    const uint8_t* pixels; uint64_t row, chan;          // chan: 0 for interleaved rows
    uint32_t w, h, chans;
    uint64_t slot;                                      // offset of its slot in d_out
};

// Enqueues the ragged pipeline for images im[k] (k in `ids`), all bound for the 16-pixel kernels.  Caller holds ctx.mu.
//
// Launches: per non-empty (chans, loader) class a scan and a pack kernel (and a hist kernel in 2-pass mode), then one launch each of
// the per-image kernels -- offsets, Adler-32, scanline-CRC combine, stored-only stream CRC (and the Huffman build in 2-pass mode).
static int encode_ragged_locked(Context& c, const std::vector<RaggedImage>& im, const std::vector<uint32_t>& ids, uint32_t flags,
                                uint8_t* d_out, uint32_t* d_sizes, cudaStream_t s, uint8_t* stage)
{
    const uint32_t m = (uint32_t)ids.size();
    const bool two_pass = (flags & FPNGB_ENCODE_SLOWER) && !(flags & FPNGB_FORCE_UNCOMPRESSED);
    size_t rows = 0, lanes = 0;
    for (uint32_t k : ids) { rows += im[k].h; lanes += (size_t)im[k].h * (((im[k].w + 511u) / 512u) * 32u); }
    const uint32_t rpw = pack16_rows_per_warp(rows), scan_rows = scan16_rows_per_cta();
    // class of an image: (chans == 4) * 3 + loader, the loader by the uniform launch's rule for one image
    constexpr int kClasses = 6;
    std::vector<uint32_t> cls(m);
    uint32_t cls_count[kClasses] = {0};
    for (uint32_t j = 0; j < m; j++) {
        const RaggedImage& r = im[ids[j]];
        const int load = r.chan ? kLoad16Planar : walk16_eligible(r.pixels, 0, (uint32_t)r.row, r.w, r.chans) ? kLoad16Staged : kLoad16Direct;
        cls[j] = (r.chans == 4 ? 3u : 0u) + (uint32_t)load;
        cls_count[cls[j]]++;
    }

    // workspace: exact, sum(h) scanlines and sum(h * lane pitch) lane records, then the descriptor table and the work lists
    const size_t table = align_up((size_t)m * sizeof(ImageDesc), 16) + (size_t)m * 5 * 4;
    size_t o = 0;
    const size_t o_bits = o; o = align_up(o + rows * 4, 256);
    const size_t o_adl = o; o = align_up(o + rows * 8, 256);
    const size_t o_ofs = o; o = align_up(o + rows * 8, 256);
    const size_t o_rcrc = o; o = align_up(o + rows * 4, 256);
    const size_t o_st = o; o = align_up(o + (size_t)m * sizeof(ImageState), 256);
    const size_t o_hist = o; o = align_up(o + (two_pass ? (size_t)m * 288 * 4 : 0), 256);
    const size_t o_books = o; o = align_up(o + (two_pass ? (size_t)m * sizeof(CodeBook) : 0), 256);
    const size_t o_lane = o; o = align_up(o + lanes * 8, 256);
    const size_t o_table = o; o = align_up(o + table, 256);
    int rc = c.ws.reserve(o);
    if (rc) return rc;
    rc = c.ws_acquire(s);
    if (rc) return rc;
    uint8_t* b = (uint8_t*)c.ws.p;
    uint32_t* row_bits = (uint32_t*)(b + o_bits); uint2* row_adler = (uint2*)(b + o_adl);
    unsigned long long* row_ofs = (unsigned long long*)(b + o_ofs); uint32_t* row_crc = (uint32_t*)(b + o_rcrc);
    ImageState* st = (ImageState*)(b + o_st); uint32_t* hist = (uint32_t*)(b + o_hist); CodeBook* books = (CodeBook*)(b + o_books);
    uint2* lane_ofs = (uint2*)(b + o_lane);
    const ImageDesc* d_desc = (const ImageDesc*)(b + o_table);

    // the table in staging: ImageDesc[m] | per class, in class order: img[], scan CTA prefix[], pack CTA prefix[] | crc img[], crc prefix[]
    ImageDesc* desc = (ImageDesc*)stage;
    uint32_t* lists = (uint32_t*)(stage + align_up((size_t)m * sizeof(ImageDesc), 16));
    uint32_t* l_img = lists; uint32_t* l_scan = lists + m; uint32_t* l_pack = lists + 2 * m; uint32_t* l_crc_img = lists + 3 * m; uint32_t* l_crc = lists + 4 * m;
    uint32_t cls_first[kClasses], fill[kClasses];
    for (int k = 0, acc = 0; k < kClasses; k++) { cls_first[k] = fill[k] = acc; acc += cls_count[k]; }
    uint64_t cls_scan_ctas[kClasses] = {0}, cls_pack_ctas[kClasses] = {0}, crc_ctas = 0;
    size_t row_base = 0, lane_base = 0;
    uint32_t max_split = 1;
    for (uint32_t j = 0; j < m; j++) {
        const RaggedImage& r = im[ids[j]];
        ImageDesc& d = desc[j];
        memset(&d, 0, sizeof d);
        d.pixels = r.pixels; d.chan_stride = r.chan; d.row_base = row_base; d.lane_base = lane_base; d.out_ofs = r.slot;
        d.book = two_pass ? books + j : c.d_static_books + (r.chans == 4 ? 1 : 0);
        d.row_pitch = (uint32_t)r.row; d.w = r.w; d.h = r.h; d.chans = r.chans; d.lane_pitch = ((r.w + 511u) / 512u) * 32u; d.index = ids[j];
        make_png_header(d.png_header, r.w, r.h, r.chans);
        row_base += r.h; lane_base += (size_t)r.h * d.lane_pitch;
        const uint32_t k = cls[j], q = fill[k]++;
        l_img[q] = j;
        l_scan[q] = (uint32_t)cls_scan_ctas[k]; cls_scan_ctas[k] += (r.h + scan_rows - 1) / scan_rows;
        const uint32_t pack_rows = pack16_rows_per_cta(rpw, r.chans);
        l_pack[q] = (uint32_t)cls_pack_ctas[k]; cls_pack_ctas[k] += (r.h + pack_rows - 1) / pack_rows;
        l_crc_img[j] = j; l_crc[j] = (uint32_t)crc_ctas; crc_ctas += crc_stream_ctas_for(max_encoded_size(r.w, r.h, r.chans));
        max_split = std::max(max_split, row_crc_split_for(r.h));
    }
    for (int k = 0; k < kClasses; k++) if (cls_scan_ctas[k] > 0x7FFFFFFFull || cls_pack_ctas[k] > 0x7FFFFFFFull) return FPNGB_ERR_INVALID_ARG;
    if (crc_ctas > 0x7FFFFFFFull) return FPNGB_ERR_INVALID_ARG;
    FPNGB_CUDA_OK(cudaMemcpyAsync((void*)d_desc, stage, table, cudaMemcpyHostToDevice, s));
    const uint32_t* d_lists = (const uint32_t*)((const uint8_t*)d_desc + align_up((size_t)m * sizeof(ImageDesc), 16));
    auto work = [&](int k, int list) {                 // list 1: scan prefix, 2: pack prefix
        return RaggedWork{d_desc, d_lists + cls_first[k], d_lists + (size_t)list * m + cls_first[k], cls_count[k]};
    };
    if (g_profile) g_prof_call++;
    ProfSet* ps = prof_begin(s);

    // RGBA 1-pass under a table whose one-pixel-match rule can fire: the launchers take the RGBA classes' LIT1 kernels
    const uint32_t lit1_rule = (!two_pass && c.h_static_books[1].lit1_rule) ? 1u : 0u;
    RaggedParams<ScanParams> sp{};
    sp.row_bits = row_bits; sp.row_adler = row_adler; sp.st = st; sp.hist = hist; sp.lane_ofs = lane_ofs;
    sp.merge_first_unit = 0u; sp.lit1_rule = lit1_rule;
    if (two_pass) {
        FPNGB_CUDA_OK(cudaMemsetAsync(hist, 0, (size_t)m * 288 * 4, s));
        for (int k = 0; k < kClasses; k++) {
            if (!cls_count[k]) continue;
            sp.ragged = work(k, 1);
            launch_hist16_ragged(sp, (uint32_t)cls_scan_ctas[k], k >= 3 ? 4u : 3u, k % 3, s);
            count_launch(1);
        }
        prof_mark(ps, kProfHist, s);
        HuffParams hp{hist, books, 0u, 0u, d_desc};
        launch_huffman_build_ragged(hp, m, s);
        count_launch(1);
        prof_mark(ps, kProfHuff, s);
    }
    for (int k = 0; k < kClasses; k++) {
        if (!cls_count[k]) continue;
        sp.ragged = work(k, 1);
        sp.merge_first_unit = (!two_pass && k < 3) ? 1u : 0u;           // RGB 1-pass
        launch_scan16_ragged(sp, (uint32_t)cls_scan_ctas[k], k >= 3 ? 4u : 3u, k % 3, s);
        count_launch(1);
    }
    prof_mark(ps, kProfScan, s);
    OffsetsParams op{};
    op.row_bits = row_bits; op.row_ofs = row_ofs; op.st = st; op.out = d_out; op.sizes = d_sizes; op.flags = flags; op.desc = d_desc;
    launch_offsets_ragged(op, m, s);
    count_launch(1);
    prof_mark(ps, kProfOffsets, s);
    RaggedParams<PackParams> pp{};
    pp.row_ofs = row_ofs; pp.row_bits = row_bits; pp.lane_ofs = lane_ofs; pp.row_adler = row_adler; pp.st = st; pp.out = d_out;
    pp.row_crc = row_crc; pp.crc_f128b = c.crc_f128b; pp.crc_lane_mul = c.crc_lane_mul; pp.lit1_rule = lit1_rule;
    for (int k = 0; k < kClasses; k++) {
        if (!cls_count[k]) continue;
        pp.ragged = work(k, 2);
        launch_pack16_ragged(pp, (uint32_t)cls_pack_ctas[k], k >= 3 ? 4u : 3u, k % 3, rpw, s);
        count_launch(1);
    }
    prof_mark(ps, kProfPack, s);
    AdlerParams ap{row_adler, st, d_out, 0, 0, 0, 0, d_desc};
    launch_adler_finalize_ragged(ap, m, s);
    count_launch(1);
    prof_mark(ps, kProfAdler, s);
    RowCrcParams rp{row_crc, row_ofs, row_bits, nullptr, 0, st, d_out, 0, 0, d_desc};
    launch_row_crc_combine_ragged(rp, m, max_split, s);
    RaggedParams<CrcParams> cp{};
    cp.out = d_out; cp.st = st; cp.stored_only = 1u;
    cp.ragged = RaggedWork{d_desc, d_lists + 3 * (size_t)m, d_lists + 4 * (size_t)m, m};
    launch_crc_stream_ragged(cp, (uint32_t)crc_ctas, s);
    count_launch(2);
    prof_mark(ps, kProfCrc, s);
    FPNGB_CUDA_OK(cudaGetLastError());
    return c.ws_release(s);
}

// ---------------------------------------------------------------------------------------------------------
// PNG encode of the images fpng does not write (fpngb_encode_png_ragged_device): gray, gray+alpha and 16-bit.
// ---------------------------------------------------------------------------------------------------------
// The 41-byte container header of these files: signature, IHDR (depth 8 or 16, color type 0, 4, 2 or 6), and the IDAT length
// (patched per image on the device) and type.
static void make_png_enc_header(uint8_t* hdr, uint32_t w, uint32_t h, uint32_t chans, uint32_t depth)
{
    static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};
    static const uint8_t color_type[4] = {0, 4, 2, 6};
    memset(hdr, 0, kPngEncHeaderSize);
    memcpy(hdr, sig, 8);
    hdr[11] = 13; memcpy(hdr + 12, "IHDR", 4);
    for (int i = 0; i < 4; i++) { hdr[16 + i] = (uint8_t)(w >> (24 - 8 * i)); hdr[20 + i] = (uint8_t)(h >> (24 - 8 * i)); }
    hdr[24] = (uint8_t)depth; hdr[25] = color_type[chans - 1];
    const uint32_t c = host_crc32(hdr + 12, 17, 0);
    for (int i = 0; i < 4; i++) hdr[29 + i] = (uint8_t)(c >> (24 - 8 * i));
    memcpy(hdr + 37, "IDAT", 4);
}

// the (bytes per pixel, depth) classes of the PNG row kernels: gray8, GA8, gray16, GA16, RGB16, RGBA16, and in LZ77 mode only
// RGB8 and RGBA8
constexpr int kPngClasses = 8;
static const uint32_t kPngClassBpp[kPngClasses] = {1, 2, 2, 4, 6, 8, 3, 4}, kPngClassDepth[kPngClasses] = {8, 8, 16, 16, 16, 16, 8, 8};
static int png_class(uint32_t bpp, uint32_t depth)
{
    for (int k = 0; k < kPngClasses; k++) if (kPngClassBpp[k] == bpp && kPngClassDepth[k] == depth) return k;
    return -1;
}

// bytes of the descriptor table, work lists and container headers (hdr_bytes in all) encode_png_locked stages for m images
static size_t png_table_bytes(size_t m, size_t hdr_bytes) { return align_up(m * sizeof(ImageDesc), 16) + m * 5 * 4 + hdr_bytes; }

// LZ77 mode (FPNGB_LZ77_CHAIN): the chain depth K of the flags, 0 when the mode is off
static uint32_t lz77_chain(uint32_t flags) { return (flags >> 16) & 0x1FFu; }
// the chain bits hold at most 256, and the mode writes no fpng file, so FPNGB_ENCODE_SLOWER has no meaning in it
static bool lz77_flags_ok(uint32_t flags)
{
    const uint32_t k = lz77_chain(flags);
    return k <= 256 && !(k && (flags & FPNGB_ENCODE_SLOWER));
}
constexpr uint32_t kLz77FlagBits = 0x1FFu << 16;

// Enqueues the PNG pipeline for images im[k] (k in `ids`, depth[k] bits per sample) into their slots.  Caller holds ctx.mu.
// Launches: per non-empty (bytes per pixel, depth) class a filter/histogram, a row-size and a pack kernel, then four per-image
// kernels: Huffman build, offsets, Adler-32, stream CRC.  own_call: no fpng pipeline ran in this call (a new profile call).
// With a chain depth in flags (LZ77 mode): per class a filter pass into S and a stored-row pass, and per call the match kernel
// and two segment kernels (bits, pack) in place of the row-size and pack kernels; the workspace adds S, its tokens (2 bytes per
// byte of S) and 16 bytes per segment.
// hdrs: the container header of image k is (*hdrs)[k] (a label map's, with PLTE / tRNS), or the 41-byte make_png_enc_header
// one when hdrs is null; d_bad: the label pre-pass's per-image flags (size 0 for a flagged image), or null.
static int encode_png_locked(Context& c, const std::vector<RaggedImage>& im, const std::vector<uint32_t>& depth, const std::vector<uint32_t>& ids,
                             uint32_t flags, uint8_t* d_out, uint32_t* d_sizes, cudaStream_t s, uint8_t* stage, bool own_call,
                             const std::vector<std::vector<uint8_t>>* hdrs = nullptr, const uint32_t* d_bad = nullptr)
{
    const uint32_t m = (uint32_t)ids.size();
    const uint32_t rpc = png_rows_per_cta();
    const uint32_t chain = lz77_chain(flags);
    size_t rows = 0;
    uint64_t s_bytes = 0, segs = 0;                                           // LZ77 mode: S and its segments
    std::vector<int> cls(m);
    uint32_t cls_count[kPngClasses] = {0};
    for (uint32_t j = 0; j < m; j++) {
        const RaggedImage& r = im[ids[j]];
        rows += r.h;
        cls[j] = png_class(r.chans * depth[ids[j]] / 8, depth[ids[j]]);
        cls_count[cls[j]]++;
        if (chain) {
            const uint64_t N = ((uint64_t)r.w * (r.chans * depth[ids[j]] / 8) + 1) * r.h;
            s_bytes += align_up(N, 16); segs += (N + kLzSegment - 1) / kLzSegment;
        }
    }
    if (segs > 0x7FFFFFFFull) return FPNGB_ERR_INVALID_ARG;
    size_t hdr_bytes = 0;
    for (uint32_t k : ids) hdr_bytes += hdrs ? (*hdrs)[k].size() : kPngEncHeaderSize;
    const size_t table = png_table_bytes(m, hdr_bytes);
    size_t o = 0;
    const size_t o_bits = o; o = align_up(o + rows * 4, 256);
    const size_t o_ofs = o; o = align_up(o + rows * 8, 256);
    const size_t o_adl = o; o = align_up(o + rows * 8, 256);
    const size_t o_filt = o; o = align_up(o + rows, 256);
    const size_t o_st = o; o = align_up(o + (size_t)m * sizeof(ImageState), 256);
    const size_t o_hist = o; o = align_up(o + (size_t)m * 288 * 4, 256);
    const size_t o_books = o; o = align_up(o + (size_t)m * sizeof(CodeBook), 256);
    const size_t o_table = o; o = align_up(o + table, 256);
    const size_t o_s = o; o = align_up(o + s_bytes, 256);
    const size_t o_tok = o; o = align_up(o + 2 * s_bytes, 256);
    const size_t o_segu = o; o = align_up(o + segs * 4, 256);
    const size_t o_segb = o; o = align_up(o + segs * 4, 256);
    const size_t o_sego = o; o = align_up(o + segs * 8, 256);
    const size_t o_dhist = o; o = align_up(o + (chain ? (size_t)m * 32 * 4 : 0), 256);
    int rc = c.ws.reserve(o);
    if (rc) return rc;
    rc = c.ws_acquire(s);
    if (rc) return rc;
    uint8_t* b = (uint8_t*)c.ws.p;
    PngEncParams p{};
    p.row_bits = (uint32_t*)(b + o_bits); p.row_ofs = (unsigned long long*)(b + o_ofs); p.row_adler = (uint2*)(b + o_adl);
    p.row_filter = b + o_filt; p.st = (ImageState*)(b + o_st); p.hist = (uint32_t*)(b + o_hist);
    CodeBook* books = (CodeBook*)(b + o_books);
    const ImageDesc* d_desc = (const ImageDesc*)(b + o_table);
    const size_t lists_at = align_up((size_t)m * sizeof(ImageDesc), 16), hdr_at = lists_at + (size_t)m * 5 * 4;
    p.out = d_out; p.sizes = d_sizes; p.flags = flags; p.desc = d_desc; p.headers = (const uint8_t*)d_desc + hdr_at; p.bad = d_bad;

    // the table in staging: ImageDesc[m] | row-kernel img[] and CTA prefix[] per class, in class order | crc img[], crc prefix[] |
    // LZ77 segment prefix[] | the container headers
    ImageDesc* desc = (ImageDesc*)stage;
    uint32_t* lists = (uint32_t*)(stage + lists_at);
    uint32_t* l_img = lists; uint32_t* l_cta = lists + m; uint32_t* l_crc_img = lists + 2 * m; uint32_t* l_crc = lists + 3 * m;
    uint32_t* l_seg = lists + 4 * m;
    uint64_t s_fill = 0, seg_fill = 0;
    uint8_t* headers = stage + hdr_at;
    uint32_t hdr_fill = 0;
    uint32_t cls_first[kPngClasses], fill[kPngClasses];
    for (int k = 0, acc = 0; k < kPngClasses; k++) { cls_first[k] = fill[k] = acc; acc += cls_count[k]; }
    uint64_t cls_ctas[kPngClasses] = {0}, crc_ctas = 0;
    size_t row_base = 0;
    for (uint32_t j = 0; j < m; j++) {
        const RaggedImage& r = im[ids[j]];
        const uint32_t bpp = r.chans * depth[ids[j]] / 8;
        ImageDesc& d = desc[j];
        memset(&d, 0, sizeof d);
        d.pixels = r.pixels; d.chan_stride = r.chan; d.row_base = row_base; d.out_ofs = r.slot; d.book = books + j;
        d.row_pitch = (uint32_t)r.row; d.w = r.w; d.h = r.h; d.chans = bpp; d.index = ids[j];
        d.hdr_at = hdr_fill;
        if (hdrs) {
            const std::vector<uint8_t>& hv = (*hdrs)[ids[j]];
            memcpy(headers + hdr_fill, hv.data(), hv.size());
            d.hdr_len = (uint32_t)hv.size();
        } else {
            make_png_enc_header(headers + hdr_fill, r.w, r.h, r.chans, depth[ids[j]]);
            d.hdr_len = kPngEncHeaderSize;
        }
        hdr_fill += d.hdr_len;
        row_base += r.h;
        const uint64_t N = ((uint64_t)r.w * bpp + 1) * r.h;
        d.lz_ofs = s_fill; d.seg_base = seg_fill; d.nseg = (uint32_t)((N + kLzSegment - 1) / kLzSegment);
        l_seg[j] = (uint32_t)seg_fill;
        if (chain) { s_fill += align_up(N, 16); seg_fill += d.nseg; }
        const int k = cls[j];
        const uint32_t q = fill[k]++;
        l_img[q] = j; l_cta[q] = (uint32_t)cls_ctas[k]; cls_ctas[k] += (r.h + rpc - 1) / rpc;
        l_crc_img[j] = j; l_crc[j] = (uint32_t)crc_ctas;
        crc_ctas += crc_stream_ctas_for(max_encoded_size(r.w, r.h, bpp) + (d.hdr_len - kPngEncHeaderSize));
    }
    for (int k = 0; k < kPngClasses; k++) if (cls_ctas[k] > 0x7FFFFFFFull) return FPNGB_ERR_INVALID_ARG;
    if (crc_ctas > 0x7FFFFFFFull) return FPNGB_ERR_INVALID_ARG;
    FPNGB_CUDA_OK(cudaMemcpyAsync((void*)d_desc, stage, table, cudaMemcpyHostToDevice, s));
    const uint32_t* d_lists = (const uint32_t*)((const uint8_t*)d_desc + lists_at);
    if (g_profile && own_call) g_prof_call++;
    ProfSet* ps = prof_begin(s);
    uint64_t launches = 0;
    auto rows_pass = [&](int mode) {
        for (int k = 0; k < kPngClasses; k++) {
            if (!cls_count[k]) continue;
            p.ragged = RaggedWork{d_desc, d_lists + cls_first[k], d_lists + m + cls_first[k], cls_count[k]};
            launch_png_rows(p, (uint32_t)cls_ctas[k], kPngClassBpp[k], kPngClassDepth[k], mode, s);
            launches++;
        }
    };

    FPNGB_CUDA_OK(cudaMemsetAsync(p.hist, 0, (size_t)m * 288 * 4, s));
    if (chain) {
        PngLzParams q{p};
        q.lz_s = b + o_s; q.lz_tok = (uint16_t*)(b + o_tok); q.seg_units = (uint32_t*)(b + o_segu); q.seg_bits = (uint32_t*)(b + o_segb);
        q.seg_ofs = (unsigned long long*)(b + o_sego); q.dhist = (uint32_t*)(b + o_dhist); q.chain = chain;
        auto lz_rows_pass = [&](int mode) {
            for (int k = 0; k < kPngClasses; k++) {
                if (!cls_count[k]) continue;
                q.ragged = RaggedWork{d_desc, d_lists + cls_first[k], d_lists + m + cls_first[k], cls_count[k]};
                launch_png_lz_rows(q, (uint32_t)cls_ctas[k], kPngClassBpp[k], kPngClassDepth[k], mode, s);
                launches++;
            }
        };
        FPNGB_CUDA_OK(cudaMemsetAsync(q.dhist, 0, (size_t)m * 32 * 4, s));
        lz_rows_pass(0);
        prof_mark(ps, kProfHist, s);
        q.ragged = RaggedWork{d_desc, d_lists + 2 * (size_t)m, d_lists + 4 * (size_t)m, m};    // one CTA per segment
        launch_lz_match(q, (uint32_t)segs, s);
        prof_mark(ps, kProfMatch, s);
        HuffParams hp{p.hist, books, 0u, 0u, d_desc, q.dhist};
        launch_huffman_build_lz(hp, m, s);
        prof_mark(ps, kProfHuff, s);
        launch_lz_segments(q, (uint32_t)segs, false, s);
        prof_mark(ps, kProfScan, s);
        launch_png_lz_offsets(q, m, s);
        prof_mark(ps, kProfOffsets, s);
        launch_lz_segments(q, (uint32_t)segs, true, s);
        lz_rows_pass(1);
        prof_mark(ps, kProfPack, s);
        launches += 3;
    } else {
        rows_pass(0);
        prof_mark(ps, kProfHist, s);
        HuffParams hp{p.hist, books, 0u, 0u, d_desc};
        launch_huffman_build_png(hp, m, s);
        prof_mark(ps, kProfHuff, s);
        rows_pass(1);
        prof_mark(ps, kProfScan, s);
        launch_png_offsets(p, m, s);
        prof_mark(ps, kProfOffsets, s);
        rows_pass(2);
        prof_mark(ps, kProfPack, s);
    }
    AdlerParams ap{p.row_adler, p.st, d_out, 0, 0, 0, 0, d_desc};
    launch_adler_finalize_png(ap, m, s);
    prof_mark(ps, kProfAdler, s);
    RaggedParams<CrcParams> cp{};
    cp.out = d_out; cp.st = p.st; cp.stored_only = 0u;
    cp.ragged = RaggedWork{d_desc, d_lists + 2 * (size_t)m, d_lists + 3 * (size_t)m, m};
    launch_crc_stream_png(cp, (uint32_t)crc_ctas, s);
    prof_mark(ps, kProfCrc, s);
    count_launch(launches + 4);
    FPNGB_CUDA_OK(cudaGetLastError());
    return c.ws_release(s);
}

}  // namespace fpngb

using namespace fpngb;

// ---------------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------------
extern "C" {

int fpngb_init(int device)
{
    std::lock_guard<std::mutex> lk(g_init_mu);
    if (g_ctx.ready) return FPNGB_OK;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) return FPNGB_ERR_NO_DEVICE;
    if (device < 0) { if (cudaGetDevice(&device) != cudaSuccess) return FPNGB_ERR_NO_DEVICE; }
    if (device >= count) return FPNGB_ERR_INVALID_ARG;
    FPNGB_CUDA_OK(cudaSetDevice(device));
    Context& c = g_ctx;
    c.device = device;
    FPNGB_CUDA_OK(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
    if (!build_static_book(c.h_static_books[0], kStaticHdrRGB, sizeof kStaticHdrRGB, kStaticHdrRGBTail, kStaticHdrRGBTailBits, 3)) return FPNGB_ERR_INTERNAL;
    if (!build_static_book(c.h_static_books[1], kStaticHdrRGBA, sizeof kStaticHdrRGBA, kStaticHdrRGBATail, kStaticHdrRGBATailBits, 4)) return FPNGB_ERR_INTERNAL;
    FPNGB_CUDA_OK(cudaMalloc(&c.d_static_books, 2 * sizeof(CodeBook)));
    FPNGB_CUDA_OK(cudaMemcpy(c.d_static_books, c.h_static_books, 2 * sizeof(CodeBook), cudaMemcpyHostToDevice));
    int rc = fused_tables_init();
    if (rc) return rc;
    rc = crc_stream_tables_init();
    if (rc) return rc;
    rc = crc_stream_table_ptrs(&c.crc_f128b, &c.crc_lane_mul);
    if (rc) return rc;
    c.pin_small.pinned = true;
    rc = c.pin_small.reserve(1 << 16);
    if (rc) return rc;
    c.ready = true;
    return FPNGB_OK;
}

int fpngb_is_initialized(void) { return g_ctx.ready ? 1 : 0; }
const char* fpngb_version(void) { return "fpng_b200 0.1 (sm_90a; format-compatible with fpng 1.0.6)"; }
uint64_t fpngb_launch_count(void) { return g_launches.load(); }

size_t fpngb_max_encoded_size(uint32_t w, uint32_t h, uint32_t chans) { return max_encoded_size(w, h, chans); }

// test hook: scanlines per warp of the 16-pixel scan/pack kernels (0 = automatic); not part of the reference surface
FPNGB_API void fpngb_debug_rows_per_warp(uint32_t v) { set_rows_per_warp16(v); }

// test hook: 1 = the single-pass encoder where it applies; any other value (the tests restore the default with -1) = the two-kernel
// encoder; not part of the reference surface
FPNGB_API void fpngb_debug_use_fused(int mode) { g_fused = mode == 1; }
FPNGB_API void fpngb_debug_crc_overlap(int on) { g_crc_overlap = on != 0; }
// test hook: 0 = the two-kernel encoder leaves the IDAT CRC to the file-reading CRC kernel instead of computing it in the pack kernel
FPNGB_API void fpngb_debug_pack_crc(int on) { g_pack_crc = on != 0; }

// exposes the static code books to the tests (sizes[288], codes[288]); not part of the reference surface
FPNGB_API int fpngb_debug_static_table(uint32_t chans, uint8_t* sizes, uint16_t* codes, uint32_t* hdr_bits)
{
    CodeBook cb;
    const bool ok = chans == 3 ? build_static_book(cb, kStaticHdrRGB, sizeof kStaticHdrRGB, kStaticHdrRGBTail, kStaticHdrRGBTailBits, 3)
                               : build_static_book(cb, kStaticHdrRGBA, sizeof kStaticHdrRGBA, kStaticHdrRGBATail, kStaticHdrRGBATailBits, 4);
    if (!ok) return FPNGB_ERR_INTERNAL;
    memcpy(sizes, cb.sym_size, 288);
    for (int i = 0; i < 256; i++) codes[i] = (uint16_t)(cb.lit[i] & 0xFFFF);
    for (int i = 256; i < 288; i++) codes[i] = 0;
    codes[256] = (uint16_t)(cb.eob & 0xFFFF);
    *hdr_bits = cb.hdr_bits;
    return FPNGB_OK;
}

// Body of fpngb_encode_batch_device_strided (typed false, fmt unused) and fpngb_encode_batch_device_typed (fmt required).
static int encode_batch_impl(const void* d_pixels, size_t image_stride, size_t row_pitch, size_t pixel_stride, size_t chan_stride, uint32_t n,
                             uint32_t w, uint32_t h, uint32_t chans, bool typed, const fpngb_pixel_format* fmt, uint32_t flags, void* d_out,
                             size_t out_stride, uint32_t* d_sizes, void* stream)
{
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    PixelFormat f = uint8_format();
    if (typed) { const int rc = parse_format(fmt, chans, f); if (rc) return rc; }
    if (!d_pixels || !d_out || !d_sizes || n == 0 || n > 65535 || !valid_dims(w, h, chans)) return FPNGB_ERR_INVALID_ARG;
    // any interleaved or planar layout, overlapping ones included (the pixels are only read)
    Layout L;
    const int rc = check_layout(d_pixels, image_stride, row_pitch, pixel_stride, chan_stride, n, h, w, chans, f.elem, false, L);
    if (rc) return rc;
    if (!typed && L.row > 0xFFFFFFFFull) return FPNGB_ERR_INVALID_ARG;      // the uint8 kernels take a 32-bit row pitch
    if (out_stride < max_encoded_size(w, h, chans)) return FPNGB_ERR_BUFFER_TOO_SMALL;
    if (out_stride % 16 || (uintptr_t)d_out % 16) return FPNGB_ERR_ALIGNMENT;
    Context& c = g_ctx;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    cudaStream_t s = (cudaStream_t)stream;      // NULL = the CUDA default stream, exactly as the caller passed it
    return encode_batch_locked(c, (const uint8_t*)d_pixels, L, f, n, w, h, chans, flags, (uint8_t*)d_out, out_stride, d_sizes, s);
}

int fpngb_encode_batch_device_strided(const void* d_pixels, size_t image_stride, size_t row_pitch, size_t pixel_stride, size_t chan_stride,
                                      uint32_t n, uint32_t w, uint32_t h, uint32_t chans, uint32_t flags, void* d_out, size_t out_stride,
                                      uint32_t* d_sizes, void* stream)
{
    return encode_batch_impl(d_pixels, image_stride, row_pitch, pixel_stride, chan_stride, n, w, h, chans, false, nullptr, flags, d_out,
                             out_stride, d_sizes, stream);
}

int fpngb_encode_batch_device_typed(const void* d_pixels, size_t image_stride, size_t row_pitch, size_t pixel_stride, size_t chan_stride,
                                    uint32_t n, uint32_t w, uint32_t h, uint32_t chans, const fpngb_pixel_format* fmt, uint32_t flags,
                                    void* d_out, size_t out_stride, uint32_t* d_sizes, void* stream)
{
    return encode_batch_impl(d_pixels, image_stride, row_pitch, pixel_stride, chan_stride, n, w, h, chans, true, fmt, flags, d_out,
                             out_stride, d_sizes, stream);
}

int fpngb_encode_batch_device(const void* d_pixels, size_t image_stride, uint32_t n, uint32_t w, uint32_t h, uint32_t chans,
                              uint32_t flags, void* d_out, size_t out_stride, uint32_t* d_sizes, void* stream)
{
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!d_pixels || !d_out || !d_sizes || n == 0 || !valid_dims(w, h, chans)) return FPNGB_ERR_INVALID_ARG;
    if (image_stride < (size_t)w * h * chans) return FPNGB_ERR_INVALID_ARG;
    return fpngb_encode_batch_device_strided(d_pixels, image_stride, (size_t)w * chans, chans, 1, n, w, h, chans, flags, d_out, out_stride,
                                             d_sizes, stream);
}

static size_t reduced_bound(uint32_t w, uint32_t h, uint32_t chans, uint32_t depth);
static int reduce_images_locked(Context& c, std::vector<RaggedImage>& im, const std::vector<Layout>& src, std::vector<uint32_t>& depth,
                                cudaStream_t s, std::vector<std::vector<uint8_t>>& hdrs, std::vector<ReduceConvDesc>& conv,
                                std::vector<uint32_t>& conv_img, uint64_t& conv_bytes);

// Body of the ragged encode calls: fpngb_encode_png_ragged_device and fpngb_encode_ragged_device (typed false, fmt unused) and their
// _typed twins (fmt required), with dims n x {w, h, chans, depth}.  Images of depth 8 with 3 or 4 channels take fpng's route, the
// others encode_png_locked.  A typed call first converts every image in one launch into tight rows of its output depth in c.conv;
// from there on it is the untyped call on those rows.  The conversion and both routes sit inside one workspace bracket
// (ws_acquire ... the last ws_release), so a call on another stream cannot overwrite c.conv before this call's kernels have read it.
// reduce (FPNGB_ENCODE_REDUCE, untyped only): reduce_images_locked first picks each image's format, waiting once on the host, and
// rewrites the images whose format changed as reduced rows in c.conv; the routes then take every image in its reduced format.
static int encode_images_impl(uint32_t n, const uint64_t* pixels, const uint32_t* dims, const uint64_t* strides, bool typed,
                              const fpngb_pixel_format* fmt, uint32_t flags, void* d_out, size_t out_cap, uint64_t* d_out_offsets,
                              uint32_t* d_sizes, void* stream, bool reduce = false)
{
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (n == 0 || n > 65535 || !pixels || !dims || !d_out || !d_out_offsets || !d_sizes) return FPNGB_ERR_INVALID_ARG;
    PixelFormat f = uint8_format();
    if (typed) {                                        // scale and bias are in use up to the largest channel count
        uint32_t max_chans = 0;
        for (uint32_t i = 0; i < n; i++) max_chans = std::max(max_chans, dims[4 * i + 2]);
        const int rc = parse_format(fmt, max_chans, f);
        if (rc) return rc;
    }
    std::vector<RaggedImage> im(n);
    std::vector<Layout> src(n);
    std::vector<uint32_t> depth(n), fpng_ids, png_ids;
    uint64_t total = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t w = dims[4 * i], h = dims[4 * i + 1], chans = dims[4 * i + 2], dep = dims[4 * i + 3];
        if (!pixels[i] || (dep != 8 && dep != 16) || chans < 1 || chans > 4) return FPNGB_ERR_INVALID_ARG;
        const uint32_t es = typed ? f.elem : dep / 8, bpp = chans * dep / 8;   // input element and output pixel bytes
        const bool fpng = dep == 8 && chans >= 3 && !lz77_chain(flags);  // fpng's files, as fpngb_encode_ragged_device writes them
        if (fpng ? !valid_dims(w, h, chans)
                 : (w < 1 || h < 1 || w > (1u << 24) || h > (1u << 24) || max_encoded_size(w, h, bpp) > 0x7FFFFFFFull))
            return FPNGB_ERR_INVALID_ARG;                                 // one IDAT chunk must hold the stored file
        const uint64_t bound = reduce ? reduced_bound(w, h, chans, dep) : max_encoded_size(w, h, bpp);
        if (reduce && bound > 0x7FFFFFFFull) return FPNGB_ERR_INVALID_ARG;
        const uint64_t row = strides ? strides[3 * i] : (uint64_t)w * chans * es, pixel = strides ? strides[3 * i + 1] : chans * es;
        const uint64_t chan = (strides && chans > 1) ? strides[3 * i + 2] : es;   // a single channel's stride addresses nothing
        Layout& L = src[i];
        const int rc = check_layout((const void*)(uintptr_t)pixels[i], 0, row, pixel, chan, 1, h, w, chans, es, false, L);
        if (rc) return rc;
        if (!typed && L.row > 0xFFFFFFFFull) return FPNGB_ERR_INVALID_ARG;  // the integer kernels take a 32-bit row pitch
        im[i] = RaggedImage{(const uint8_t*)(uintptr_t)pixels[i], L.row, L.planar ? L.chan : 0, w, h, chans, total};
        depth[i] = dep;
        (fpng ? fpng_ids : png_ids).push_back(i);
        total += align_up(bound, 16);
    }
    if (out_cap < total) return FPNGB_ERR_BUFFER_TOO_SMALL;
    if ((uintptr_t)d_out % 16) return FPNGB_ERR_ALIGNMENT;
    Context& c = g_ctx;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    cudaStream_t s = (cudaStream_t)stream;
    uint8_t* out = (uint8_t*)d_out;

    // reduce: the images in their reduced formats; the headers of the PNG route's images; the conversions into c.conv
    std::vector<std::vector<uint8_t>> hdrs;
    std::vector<ReduceConvDesc> rconv;
    std::vector<uint32_t> rconv_img;                                     // the image of rconv[j]
    uint64_t rconv_bytes = 0;
    size_t png_hdr_bytes = png_ids.size() * kPngEncHeaderSize;
    if (reduce) {
        flags &= ~(uint32_t)FPNGB_ENCODE_REDUCE;
        const int rc = reduce_images_locked(c, im, src, depth, s, hdrs, rconv, rconv_img, rconv_bytes);
        if (rc) { c.ws_release(s); return rc; }
        fpng_ids.clear(); png_ids.clear(); png_hdr_bytes = 0;
        for (uint32_t i = 0; i < n; i++) {
            const bool fpng = depth[i] == 8 && im[i].chans >= 3 && !lz77_chain(flags);
            (fpng ? fpng_ids : png_ids).push_back(i);
            if (!fpng) png_hdr_bytes += hdrs[i].size();
        }
    }

    // typed: the conversion buffer holds image i's tight rows (w * chans samples of depth / 8 bytes) at a 16-byte aligned offset
    // at[i], then the descriptor table at desc_at
    std::vector<uint64_t> at(typed ? n : 0);
    uint64_t desc_at = 0;
    if (typed) {
        for (uint32_t i = 0; i < n; i++) { at[i] = desc_at; desc_at += align_up((uint64_t)im[i].w * im[i].h * im[i].chans * (depth[i] / 8), 16); }
        desc_at = align_up(desc_at, 256);
        const int rc = c.conv.reserve(desc_at + (size_t)n * sizeof(ConvDesc));
        if (rc) return rc;
    }

    // staging: d_out_offsets (n + 1), then the fpng images' table and work lists, then the PNG images' table and work lists, then
    // (typed) the conversion descriptors
    const size_t ofs_bytes = align_up((size_t)(n + 1) * 8, 16);
    const size_t fpng_table = align_up(align_up(fpng_ids.size() * sizeof(ImageDesc), 16) + fpng_ids.size() * 5 * 4, 16);
    const size_t conv_stage = align_up(ofs_bytes + fpng_table + png_table_bytes(png_ids.size(), png_hdr_bytes), 16);
    StageSlot* sl = nullptr;
    int rc = c.stage_slot(conv_stage + (typed ? (size_t)n * sizeof(ConvDesc) : rconv.size() * sizeof(ReduceConvDesc)), &sl);
    if (rc) { if (reduce) c.ws_release(s); return rc; }
    uint8_t* stage = (uint8_t*)sl->buf.p;
    uint64_t* h_ofs = (uint64_t*)stage;
    for (uint32_t i = 0; i < n; i++) h_ofs[i] = im[i].slot;
    h_ofs[n] = total;
    FPNGB_CUDA_OK(cudaMemcpyAsync(d_out_offsets, h_ofs, (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, s));

    if (typed) {
        uint8_t* cb = (uint8_t*)c.conv.p;
        ConvDesc* hd = (ConvDesc*)(stage + conv_stage);
        unsigned long long ctas = 0;
        for (uint32_t i = 0; i < n; i++) {
            RaggedImage& r = im[i];
            const uint32_t ob = depth[i] / 8;
            hd[i] = conv_desc(r.pixels, src[i], 1, r.w, r.h, r.chans, at[i], ctas, ob);
            ctas += hd[i].ctas_per_image;
            r.pixels = cb + at[i]; r.row = (uint64_t)r.w * r.chans * ob; r.chan = 0;
        }
        rc = c.ws_acquire(s);
        if (rc) return rc;
        FPNGB_CUDA_OK(cudaMemcpyAsync(cb + desc_at, hd, (size_t)n * sizeof(ConvDesc), cudaMemcpyHostToDevice, s));
        // the PNG instantiations only when an image needs them: for 8-bit RGB / RGBA both write the same bytes
        convert_enqueue(hd, n, (const ConvDesc*)(cb + desc_at), f, cb, s, !png_ids.empty());
    }
    // a route that fails after the conversion still closes the bracket, so that later calls wait for the conversion
    auto fail = [&](int code) { prof_drop_conv(); if (typed || reduce) c.ws_release(s); cudaEventRecord(sl->ev, s); return code; };
    if (!rconv.empty()) {                  // the reduced rows: one launch over the images whose format changed (profile slot 9)
        const uint64_t rdesc_at = align_up(rconv_bytes, 256);
        rc = c.conv.reserve(rdesc_at + rconv.size() * sizeof(ReduceConvDesc));
        if (rc) return fail(rc);
        uint8_t* cb = (uint8_t*)c.conv.p;
        unsigned long long ctas = 0;
        for (size_t j = 0; j < rconv.size(); j++) {
            im[rconv_img[j]].pixels = cb + rconv[j].dst;
            rconv[j].cta_start = ctas; ctas += reduce_convert_ctas(rconv[j].words, rconv[j].h);
        }
        if (ctas > 0x7FFFFFFFull) return fail(FPNGB_ERR_INVALID_ARG);
        memcpy(stage + conv_stage, rconv.data(), rconv.size() * sizeof(ReduceConvDesc));
        FPNGB_CUDA_OK(cudaMemcpyAsync(cb + rdesc_at, stage + conv_stage, rconv.size() * sizeof(ReduceConvDesc), cudaMemcpyHostToDevice, s));
        ProfSet* ps = g_prof_conv;
        if (ps) cudaEventRecord(ps->conv_start, s);
        launch_reduce_convert(ReduceConvParams{(const ReduceConvDesc*)(cb + rdesc_at), (uint32_t)rconv.size(), cb}, ctas, s);
        count_launch(1);
        if (ps) prof_mark(ps, kProfConvert, s);
    }
    if (!fpng_ids.empty()) {
        rc = encode_ragged_locked(c, im, fpng_ids, flags, out, d_sizes, s, stage + ofs_bytes);
        if (rc) return fail(rc);
    }
    if (!png_ids.empty()) {
        rc = encode_png_locked(c, im, depth, png_ids, flags, out, d_sizes, s, stage + ofs_bytes + fpng_table, fpng_ids.empty(),
                               reduce ? &hdrs : nullptr);
        if (rc) return fail(rc);
    }
    prof_drop_conv();
    FPNGB_CUDA_OK(cudaEventRecord(sl->ev, s));
    return FPNGB_OK;
}

// ---- label maps (fpngb_encode_label_ragged_device) -------------------------------------------------------------------------
// tRNS length of a palette: 1 + the last entry whose alpha is not 255, 0 for an RGB palette or one that is opaque throughout
static uint32_t label_trns_len(const fpngb_label_palette* pal)
{
    uint32_t t = 0;
    if (pal && pal->entries && pal->chans == 4)
        for (uint32_t e = 0; e < pal->entries; e++) if (pal->colors[4 * e + 3] != 255) t = e + 1;
    return t;
}

// PLTE and tRNS chunk bytes of a palette (0 for a gray map)
static size_t label_chunk_bytes(const fpngb_label_palette* pal)
{
    if (!pal || !pal->entries) return 0;
    const uint32_t t = label_trns_len(pal);
    return 12 + 3 * (size_t)pal->entries + (t ? 12 + (size_t)t : 0);
}

// the rows the pre-pass writes: a gray8 image ceil(w * depth / 8) bytes wide, or for depth 16 a gray16 image w wide
static uint32_t label_packed_width(uint32_t w, uint32_t depth) { return depth == 16 ? w : (uint32_t)(((uint64_t)w * depth + 7) / 8); }

static size_t label_bound(uint32_t w, uint32_t h, uint32_t depth, const fpngb_label_palette* pal)
{
    return max_encoded_size(label_packed_width(w, depth), h, depth == 16 ? 2 : 1) + label_chunk_bytes(pal);
}

static void put_chunk(std::vector<uint8_t>& v, const char* type, const uint8_t* data, size_t len)
{
    const size_t at = v.size();
    v.resize(at + 12 + len);
    uint8_t* q = v.data() + at;
    for (int i = 0; i < 4; i++) q[i] = (uint8_t)(len >> (24 - 8 * i));
    memcpy(q + 4, type, 4);
    if (len) memcpy(q + 8, data, len);
    const uint32_t c = host_crc32(q + 4, 4 + len, 0);
    for (int i = 0; i < 4; i++) q[8 + len + i] = (uint8_t)(c >> (24 - 8 * i));
}

// signature, IHDR (depth, color type 0 or 3), PLTE and tRNS of a palette, the IDAT length (patched on the device) and type
static std::vector<uint8_t> make_label_header(uint32_t w, uint32_t h, uint32_t depth, const fpngb_label_palette* pal)
{
    uint8_t base[kPngEncHeaderSize];
    make_png_enc_header(base, w, h, 1, depth);
    std::vector<uint8_t> v(base, base + 8);
    const bool palette = pal && pal->entries;
    uint8_t ihdr[13];
    memcpy(ihdr, base + 16, 13);
    ihdr[9] = palette ? 3 : 0;
    put_chunk(v, "IHDR", ihdr, 13);
    if (palette) {
        std::vector<uint8_t> rgb(3 * (size_t)pal->entries), alpha;
        for (uint32_t e = 0; e < pal->entries; e++) for (int k = 0; k < 3; k++) rgb[3 * e + k] = pal->colors[pal->chans * e + k];
        put_chunk(v, "PLTE", rgb.data(), rgb.size());
        const uint32_t t = label_trns_len(pal);
        for (uint32_t e = 0; e < t; e++) alpha.push_back(pal->colors[4 * e + 3]);
        if (t) put_chunk(v, "tRNS", alpha.data(), t);
    }
    v.insert(v.end(), base + 33, base + kPngEncHeaderSize);
    return v;
}

size_t fpngb_max_label_encoded_size(uint32_t w, uint32_t h, uint32_t depth, const fpngb_label_palette* pal)
{
    return label_bound(w, h, depth, pal);
}

// ---- colour-type reduction (FPNGB_ENCODE_REDUCE) ---------------------------------------------------------------------------
// The largest file of any format the reduction can pick: the unreduced bound, or a depth-8 palette file with 256 entries and a
// full tRNS.  Every other candidate has at most the input's bytes per pixel (max_encoded_size grows with the row bytes).
static size_t reduced_bound(uint32_t w, uint32_t h, uint32_t chans, uint32_t depth)
{
    static const uint8_t clear[4 * 256] = {};                             // alpha 0 throughout: tRNS of 256 entries
    const fpngb_label_palette full{clear, 256, 4};
    return std::max(max_encoded_size(w, h, chans * depth / 8), label_bound(w, h, 8, &full));
}

size_t fpngb_max_reduced_encoded_size(uint32_t w, uint32_t h, uint32_t chans, uint32_t depth)
{
    if (chans < 1 || chans > 4 || (depth != 8 && depth != 16)) return 0;
    return reduced_bound(w, h, chans, depth);
}

// The formats of the rule in include/fpng_b200.h, in its tie order
enum RedFormat { kFmtGray = 0, kFmtPalette, kFmtGA, kFmtRGB, kFmtRGBA };
struct RedChoice { int fmt; uint32_t bits; uint32_t depth; };      // bits per pixel; sample depth (gray: d, or 16)

static uint32_t pil_palette_depth(uint32_t K) { return K <= 2 ? 1 : K <= 4 ? 2 : K <= 16 ? 4 : 8; }

// The format of an image of chans channels at depth bits from its analysis flags and colour count K
static RedChoice reduce_choice(uint32_t chans, uint32_t depth, uint32_t flags, uint32_t K)
{
    const bool rep8 = depth == 8 || !(flags & kRedNotRep8);
    const bool opaque = (chans & 1u) || !(flags & kRedNotOpaque);
    const bool gray = chans <= 2 || !(flags & kRedNotGray);
    const uint32_t D = rep8 ? 8 : 16;
    RedChoice best{-1, 0, 0};
    auto offer = [&](int fmt, uint32_t bits, uint32_t dep) { if (best.fmt < 0 || bits < best.bits) best = RedChoice{fmt, bits, dep}; };
    if (gray && opaque) {
        const uint32_t d = !rep8 ? 16 : !(flags & kRedNotL1) ? 1 : !(flags & kRedNotL2) ? 2 : !(flags & kRedNotL4) ? 4 : 8;
        offer(kFmtGray, d, d);
    }
    if (rep8 && !(flags & kRedOverflow)) offer(kFmtPalette, pil_palette_depth(K), pil_palette_depth(K));
    if (gray) offer(kFmtGA, 2 * D, D);
    if (opaque) offer(kFmtRGB, 3 * D, D);
    offer(kFmtRGBA, 4 * D, D);
    return best;
}

// FPNGB_ENCODE_REDUCE's analysis and decision, inside the call's workspace bracket (it opens it: ws_acquire on s).  Enqueues the
// analysis and finalise kernels (profile slot 10) over every image, reads back each image's ReduceResult and waits for it: the one
// host synchronisation of the call.  Then, per image whose format changed, rewrites im[i] / depth[i] as the rows the routes encode
// (tight rows or packed gray8 rows of a label file, words * 4 bytes apart, at byte conv_bytes of c.conv, filled by conv[j] for image
// conv_img[j] once the caller has placed them) and sets hdrs[i], the container header of every image bound for the PNG route.
static int reduce_images_locked(Context& c, std::vector<RaggedImage>& im, const std::vector<Layout>& src, std::vector<uint32_t>& depth,
                                cudaStream_t s, std::vector<std::vector<uint8_t>>& hdrs, std::vector<ReduceConvDesc>& conv,
                                std::vector<uint32_t>& conv_img, uint64_t& conv_bytes)
{
    const uint32_t n = (uint32_t)im.size();
    // c.red: ReduceState[n] | ReduceTable[n] (cleared) | ReduceResult[n] | ReduceDesc[n]
    const size_t o_tab = align_up((size_t)n * sizeof(ReduceState), 256), o_res = align_up(o_tab + (size_t)n * sizeof(ReduceTable), 256);
    const size_t o_desc = align_up(o_res + (size_t)n * sizeof(ReduceResult), 256), bytes = o_desc + (size_t)n * sizeof(ReduceDesc);
    std::vector<ReduceDesc> rd(n);
    unsigned long long ctas = 0;
    for (uint32_t i = 0; i < n; i++) {
        const RaggedImage& r = im[i];
        rd[i] = ReduceDesc{r.pixels, r.row, src[i].pixel, src[i].chan, ctas, r.w, r.h, r.chans, depth[i] / 8};
        ctas += reduce_analyze_ctas(r.w, r.h);
    }
    if (ctas > 0x7FFFFFFFull) return FPNGB_ERR_INVALID_ARG;
    int rc = c.ws_acquire(s);
    if (rc) return rc;
    rc = c.red.reserve(bytes);
    if (rc) return rc;
    StageSlot* sl = nullptr;                                              // the descriptors up, then the results down
    rc = c.stage_slot(std::max((size_t)n * sizeof(ReduceDesc), (size_t)n * sizeof(ReduceResult)), &sl);
    if (rc) return rc;
    uint8_t* b = (uint8_t*)c.red.p;
    memcpy(sl->buf.p, rd.data(), (size_t)n * sizeof(ReduceDesc));
    FPNGB_CUDA_OK(cudaMemcpyAsync(b + o_desc, sl->buf.p, (size_t)n * sizeof(ReduceDesc), cudaMemcpyHostToDevice, s));
    FPNGB_CUDA_OK(cudaMemsetAsync(b, 0, o_res, s));
    ReduceParams p{(const ReduceDesc*)(b + o_desc), n, (ReduceState*)b, (ReduceTable*)(b + o_tab), (ReduceResult*)(b + o_res)};
    prof_drop_conv();
    ProfSet* ps = g_profile ? prof_alloc() : nullptr;                      // slots 10 and 9 of the encode that follows
    if (ps) cudaEventRecord(ps->red_start, s);
    launch_reduce_analyze(p, ctas, s);
    count_launch(2);
    if (ps) { prof_mark(ps, kProfReduce, s); g_prof_conv = ps; }
    FPNGB_CUDA_OK(cudaGetLastError());
    FPNGB_CUDA_OK(cudaMemcpyAsync(sl->buf.p, b + o_res, (size_t)n * sizeof(ReduceResult), cudaMemcpyDeviceToHost, s));
    FPNGB_CUDA_OK(cudaEventRecord(sl->ev, s));
    FPNGB_CUDA_OK(cudaEventSynchronize(sl->ev));
    const ReduceResult* res = (const ReduceResult*)sl->buf.p;

    hdrs.assign(n, std::vector<uint8_t>());
    conv.clear(); conv_img.clear(); conv_bytes = 0;
    for (uint32_t i = 0; i < n; i++) {
        RaggedImage& r = im[i];
        const RedChoice ch = reduce_choice(r.chans, depth[i], res[i].flags, res[i].count);
        ReduceConvDesc d{};
        d.src = r.pixels; d.row = r.row; d.pixel = src[i].pixel; d.chan = src[i].chan;
        d.tab = p.tab + i; d.st = p.st + i; d.w = r.w; d.h = r.h; d.chans = r.chans; d.elem = depth[i] / 8;
        uint32_t out_w = r.w, out_chans = 1, out_depth = 8;
        if (ch.fmt == kFmtPalette || (ch.fmt == kFmtGray && ch.depth < 8)) {   // a label file: packed rows as a gray8 image
            d.mode = ch.fmt == kFmtPalette ? 0 : 1; d.bits = ch.depth; d.step = 255u / ((1u << ch.depth) - 1u);
            d.words = (uint32_t)(((uint64_t)r.w * ch.depth + 31) / 32);
            out_w = label_packed_width(r.w, ch.depth);
            std::vector<uint8_t> colors;
            fpngb_label_palette pal{nullptr, 0, 4};
            if (ch.fmt == kFmtPalette) {
                for (uint32_t e = 0; e < res[i].count; e++)
                    for (int k = 0; k < 4; k++) colors.push_back((uint8_t)(res[i].pal[e] >> (24 - 8 * k)));
                pal = fpngb_label_palette{colors.data(), res[i].count, 4};
            }
            hdrs[i] = make_label_header(r.w, r.h, ch.depth, ch.fmt == kFmtPalette ? &pal : nullptr);
        } else {
            out_chans = ch.fmt == kFmtGray ? 1 : ch.fmt == kFmtGA ? 2 : ch.fmt == kFmtRGB ? 3 : 4;
            out_depth = ch.depth;
            d.mode = 2; d.bits = out_chans; d.out_bytes = out_depth / 8;
            d.words = (uint32_t)(((uint64_t)r.w * out_chans * d.out_bytes + 3) / 4);
            hdrs[i].resize(kPngEncHeaderSize);                                // also read for RGB8 / RGBA8 in LZ77 mode
            make_png_enc_header(hdrs[i].data(), r.w, r.h, out_chans, out_depth);
            if (out_chans == r.chans && out_depth == depth[i]) continue;      // read in place, as without the flag
        }
        conv.push_back(d);
        conv.back().dst = conv_bytes;
        conv_img.push_back(i);
        conv_bytes += align_up((uint64_t)d.words * 4 * r.h, 16);
        r = RaggedImage{nullptr, (uint64_t)d.words * 4, 0, out_w, r.h, out_chans, r.slot};
        depth[i] = out_depth;
    }
    return FPNGB_OK;
}

// The label-map encode: call-level checks; the slots; then, in one workspace bracket, the pre-pass (label_pack_kernel) into tight
// packed rows in c.conv and encode_png_locked on those rows with each image's own header and the pre-pass's range flags.
int fpngb_encode_label_ragged_device(uint32_t n, const uint64_t* pixels, const uint32_t* dims, const uint64_t* strides,
                                     const fpngb_label_palette* palettes, uint32_t flags, void* d_out, size_t out_cap,
                                     uint64_t* d_out_offsets, uint32_t* d_sizes, void* stream)
{
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if ((flags & ~(uint32_t)(FPNGB_FORCE_UNCOMPRESSED | kLz77FlagBits)) || !lz77_flags_ok(flags)) return FPNGB_ERR_INVALID_ARG;
    if (n == 0 || n > 65535 || !pixels || !dims || !d_out || !d_out_offsets || !d_sizes) return FPNGB_ERR_INVALID_ARG;
    std::vector<RaggedImage> im(n);
    std::vector<uint32_t> depth(n), ids(n);
    std::vector<std::vector<uint8_t>> hdrs(n);
    std::vector<LabelDesc> ld(n);
    uint64_t total = 0, conv_bytes = 0, ctas = 0;
    size_t hdr_bytes = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t w = dims[4 * i], h = dims[4 * i + 1], dep = dims[4 * i + 2], elem = dims[4 * i + 3];
        const fpngb_label_palette* pal = palettes ? &palettes[i] : nullptr;
        const uint32_t K = pal ? pal->entries : 0;
        if (!pixels[i] || w < 1 || h < 1 || w > (1u << 24) || h > (1u << 24)) return FPNGB_ERR_INVALID_ARG;
        if ((elem != 1 && elem != 8) || (dep != 1 && dep != 2 && dep != 4 && dep != 8 && dep != 16) || (elem == 1 && dep > 8))
            return FPNGB_ERR_INVALID_ARG;
        if (K && (dep == 16 || !pal->colors || (pal->chans != 3 && pal->chans != 4) || K > std::min(256u, 1u << dep)))
            return FPNGB_ERR_INVALID_ARG;
        const uint64_t row = strides ? strides[2 * i] : (uint64_t)w * elem, pixel = strides ? strides[2 * i + 1] : elem;
        Layout L;
        const int rc = check_layout((const void*)(uintptr_t)pixels[i], 0, row, pixel, elem, 1, h, w, 1, elem, false, L);
        if (rc) return rc;
        const size_t bound = label_bound(w, h, dep, pal);
        if (bound > 0x7FFFFFFFull) return FPNGB_ERR_INVALID_ARG;             // one IDAT chunk must hold the stored file
        const uint32_t words = dep == 16 ? (w + 1) / 2 : (uint32_t)(((uint64_t)w * dep + 31) / 32);
        ld[i] = LabelDesc{(const uint8_t*)(uintptr_t)pixels[i], L.row, L.pixel, conv_bytes, ctas, w, h, dep,
                          K ? K : (dep == 16 ? 65536u : 1u << dep), words, i, elem, 0u};
        ctas += label_pack_ctas(words, h);
        conv_bytes += align_up((uint64_t)words * 4 * h, 16);
        im[i] = RaggedImage{nullptr, (uint64_t)words * 4, 0, label_packed_width(w, dep), h, 1, total};
        depth[i] = dep == 16 ? 16 : 8;
        ids[i] = i;
        hdrs[i] = make_label_header(w, h, dep, pal);
        hdr_bytes += hdrs[i].size();
        total += align_up(bound, 16);
    }
    if (ctas > 0x7FFFFFFFull) return FPNGB_ERR_INVALID_ARG;
    if (out_cap < total) return FPNGB_ERR_BUFFER_TOO_SMALL;
    if ((uintptr_t)d_out % 16) return FPNGB_ERR_ALIGNMENT;
    Context& c = g_ctx;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    cudaStream_t s = (cudaStream_t)stream;

    // conversion buffer: the packed rows, then the pre-pass descriptors, then the per-image range flags
    const uint64_t desc_at = align_up(conv_bytes, 256), bad_at = align_up(desc_at + (uint64_t)n * sizeof(LabelDesc), 256);
    int rc = c.conv.reserve(bad_at + (size_t)n * 4);
    if (rc) return rc;
    uint8_t* cb = (uint8_t*)c.conv.p;
    // staging: d_out_offsets (n + 1), the PNG table, the pre-pass descriptors
    const size_t ofs_bytes = align_up((size_t)(n + 1) * 8, 16);
    const size_t ld_stage = align_up(ofs_bytes + png_table_bytes(n, hdr_bytes), 16);
    StageSlot* sl = nullptr;
    rc = c.stage_slot(ld_stage + (size_t)n * sizeof(LabelDesc), &sl);
    if (rc) return rc;
    uint8_t* stage = (uint8_t*)sl->buf.p;
    uint64_t* h_ofs = (uint64_t*)stage;
    for (uint32_t i = 0; i < n; i++) { h_ofs[i] = im[i].slot; im[i].pixels = cb + ld[i].dst; }
    h_ofs[n] = total;
    memcpy(stage + ld_stage, ld.data(), (size_t)n * sizeof(LabelDesc));
    FPNGB_CUDA_OK(cudaMemcpyAsync(d_out_offsets, h_ofs, (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, s));
    rc = c.ws_acquire(s);
    if (rc) return rc;
    FPNGB_CUDA_OK(cudaMemcpyAsync(cb + desc_at, stage + ld_stage, (size_t)n * sizeof(LabelDesc), cudaMemcpyHostToDevice, s));
    uint32_t* d_bad = (uint32_t*)(cb + bad_at);
    FPNGB_CUDA_OK(cudaMemsetAsync(d_bad, 0, (size_t)n * 4, s));
    LabelPackParams lp{(const LabelDesc*)(cb + desc_at), n, cb, d_bad};
    prof_drop_conv();
    ProfSet* ps = g_profile ? prof_alloc() : nullptr;                      // slot kProfConvert of the encode that follows
    if (ps) cudaEventRecord(ps->conv_start, s);
    launch_label_pack(lp, ctas, s);
    count_launch(1);
    if (ps) { prof_mark(ps, kProfConvert, s); g_prof_conv = ps; }
    rc = encode_png_locked(c, im, depth, ids, flags, (uint8_t*)d_out, d_sizes, s, stage + ofs_bytes, true, &hdrs, d_bad);
    prof_drop_conv();
    if (rc) c.ws_release(s);                                                // later calls still wait for the pre-pass
    FPNGB_CUDA_OK(cudaEventRecord(sl->ev, s));
    return rc;
}

int fpngb_encode_png_ragged_device(uint32_t n, const uint64_t* pixels, const uint32_t* dims, const uint64_t* strides, uint32_t flags,
                                   void* d_out, size_t out_cap, uint64_t* d_out_offsets, uint32_t* d_sizes, void* stream)
{
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if ((flags & ~(uint32_t)(FPNGB_ENCODE_SLOWER | FPNGB_FORCE_UNCOMPRESSED | FPNGB_ENCODE_REDUCE | kLz77FlagBits)) || !lz77_flags_ok(flags))
        return FPNGB_ERR_INVALID_ARG;
    return encode_images_impl(n, pixels, dims, strides, false, nullptr, flags, d_out, out_cap, d_out_offsets, d_sizes, stream,
                              (flags & FPNGB_ENCODE_REDUCE) != 0);
}

int fpngb_encode_png_ragged_device_typed(uint32_t n, const uint64_t* pixels, const uint32_t* dims, const uint64_t* strides,
                                         const fpngb_pixel_format* fmt, uint32_t flags, void* d_out, size_t out_cap,
                                         uint64_t* d_out_offsets, uint32_t* d_sizes, void* stream)
{
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if ((flags & ~(uint32_t)(FPNGB_ENCODE_SLOWER | FPNGB_FORCE_UNCOMPRESSED | kLz77FlagBits)) || !lz77_flags_ok(flags))
        return FPNGB_ERR_INVALID_ARG;
    return encode_images_impl(n, pixels, dims, strides, true, fmt, flags, d_out, out_cap, d_out_offsets, d_sizes, stream);
}

// fpngb_encode_ragged_device(_typed): dims n x {w, h, chans} become {w, h, chans, 8} for fpng's 3 and 4 channels and depth 0
// otherwise, which encode_images_impl rejects at that image, after the same checks of the images before it
static int encode_ragged_fpng(uint32_t n, const uint64_t* pixels, const uint32_t* dims, const uint64_t* strides, bool typed,
                              const fpngb_pixel_format* fmt, uint32_t flags, void* d_out, size_t out_cap, uint64_t* d_out_offsets,
                              uint32_t* d_sizes, void* stream)
{
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (n == 0 || n > 65535 || !dims) return FPNGB_ERR_INVALID_ARG;
    std::vector<uint32_t> dims4(4 * (size_t)n);
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t chans = dims[3 * i + 2];
        dims4[4 * i] = dims[3 * i]; dims4[4 * i + 1] = dims[3 * i + 1]; dims4[4 * i + 2] = chans;
        dims4[4 * i + 3] = chans == 3 || chans == 4 ? 8u : 0u;
    }
    return encode_images_impl(n, pixels, dims4.data(), strides, typed, fmt, flags, d_out, out_cap, d_out_offsets, d_sizes, stream);
}

int fpngb_encode_ragged_device(uint32_t n, const uint64_t* pixels, const uint32_t* dims, const uint64_t* strides, uint32_t flags,
                               void* d_out, size_t out_cap, uint64_t* d_out_offsets, uint32_t* d_sizes, void* stream)
{
    return encode_ragged_fpng(n, pixels, dims, strides, false, nullptr, flags, d_out, out_cap, d_out_offsets, d_sizes, stream);
}

int fpngb_encode_ragged_device_typed(uint32_t n, const uint64_t* pixels, const uint32_t* dims, const uint64_t* strides,
                                     const fpngb_pixel_format* fmt, uint32_t flags, void* d_out, size_t out_cap, uint64_t* d_out_offsets,
                                     uint32_t* d_sizes, void* stream)
{
    return encode_ragged_fpng(n, pixels, dims, strides, true, fmt, flags, d_out, out_cap, d_out_offsets, d_sizes, stream);
}

int fpngb_encode_host(const void* pixels, uint32_t w, uint32_t h, uint32_t chans, uint32_t flags, void* out, size_t out_cap, size_t* out_size)
{
    if (out_size) *out_size = 0;
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!pixels || !out || !out_size || !valid_dims(w, h, chans)) return FPNGB_ERR_INVALID_ARG;
    const size_t cap = max_encoded_size(w, h, chans);
    if (out_cap < cap) return FPNGB_ERR_BUFFER_TOO_SMALL;
    Context& c = g_ctx;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    const size_t in_bytes = (size_t)w * h * chans, stride = align_up(cap, 16);
    int rc = c.dev_in.reserve(in_bytes + 64); if (rc) return rc;
    rc = c.dev_out.reserve(stride + 64); if (rc) return rc;
    uint32_t* d_size = (uint32_t*)((uint8_t*)c.dev_out.p + stride);
    cudaStream_t s = c.stream;
    FPNGB_CUDA_OK(cudaMemcpyAsync(c.dev_in.p, pixels, in_bytes, cudaMemcpyHostToDevice, s));
    rc = encode_batch_locked(c, (const uint8_t*)c.dev_in.p, tight_layout(w, chans, in_bytes), uint8_format(), 1, w, h, chans, flags,
                             (uint8_t*)c.dev_out.p, stride, d_size, s);
    if (rc) return rc;
    uint32_t* h_size = (uint32_t*)c.pin_small.p;
    FPNGB_CUDA_OK(cudaMemcpyAsync(h_size, d_size, 4, cudaMemcpyDeviceToHost, s));
    FPNGB_CUDA_OK(cudaStreamSynchronize(s));
    const size_t fsize = *h_size;
    if (fsize < kPngHeaderSize + kPngTrailerSize || fsize > cap) return FPNGB_ERR_INTERNAL;
    FPNGB_CUDA_OK(cudaMemcpyAsync(out, c.dev_out.p, fsize, cudaMemcpyDeviceToHost, s));
    FPNGB_CUDA_OK(cudaStreamSynchronize(s));
    *out_size = fsize;
    return FPNGB_OK;
}

// Pipelined host-buffer batch: chunks of the batch flow H2D -> kernels -> (sizes) -> exact-size D2H through three
// slots; chunk k+1 is enqueued before the host waits for chunk k's sizes, so copies overlap the kernels.
int fpngb_encode_batch_host(const void* pixels, size_t image_stride, uint32_t n, uint32_t w, uint32_t h, uint32_t chans,
                            uint32_t flags, void* out, size_t out_stride, uint32_t* sizes)
{
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!pixels || !out || !sizes || n == 0 || !valid_dims(w, h, chans)) return FPNGB_ERR_INVALID_ARG;
    const size_t in_bytes = (size_t)w * h * chans, cap = max_encoded_size(w, h, chans), dstride = align_up(cap, 16);
    if (image_stride < in_bytes) return FPNGB_ERR_INVALID_ARG;
    if (out_stride < cap) return FPNGB_ERR_BUFFER_TOO_SMALL;
    Context& c = g_ctx;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));

    constexpr int kSlots = 3;
    const size_t target = (size_t)64 << 20;                         // ~64 MiB of pixels per chunk
    uint32_t per_chunk = (uint32_t)(target / in_bytes); if (per_chunk < 1) per_chunk = 1; if (per_chunk > n) per_chunk = n;
    if (per_chunk > 65535u) per_chunk = 65535u;                     // grid.y limit of the batch kernels (tiny images)
    const size_t slot_in = align_up(per_chunk * in_bytes, 256), slot_out = per_chunk * dstride, slot_sz = align_up(per_chunk * 4, 256);
    int rc = c.dev_in.reserve(kSlots * slot_in); if (rc) return rc;
    rc = c.dev_out.reserve(kSlots * (slot_out + slot_sz)); if (rc) return rc;
    rc = c.pin_small.reserve(kSlots * slot_sz); if (rc) return rc;
    if (!c.copy_in) { FPNGB_CUDA_OK(cudaStreamCreateWithFlags(&c.copy_in, cudaStreamNonBlocking)); FPNGB_CUDA_OK(cudaStreamCreateWithFlags(&c.copy_out, cudaStreamNonBlocking)); }
    EventSet<4 * kSlots> evs;                                       // destroyed on every exit path
    if (!evs.ok) return FPNGB_ERR_INTERNAL;
    cudaEvent_t* ev_in = evs.ev; cudaEvent_t* ev_done = evs.ev + kSlots; cudaEvent_t* ev_sizes = evs.ev + 2 * kSlots; cudaEvent_t* ev_out = evs.ev + 3 * kSlots;
    const uint32_t nchunks = (n + per_chunk - 1) / per_chunk;
    const bool contiguous = image_stride == in_bytes;
    int result = FPNGB_OK;

    auto finish = [&](uint32_t k) -> int {      // exact-size D2H of chunk k's files
        const int sl = k % kSlots;
        const uint32_t first = k * per_chunk, cnt = (first + per_chunk <= n) ? per_chunk : n - first;
        FPNGB_CUDA_OK(cudaEventSynchronize(ev_sizes[sl]));
        const uint32_t* hs = (const uint32_t*)((uint8_t*)c.pin_small.p + sl * slot_sz);
        const uint8_t* dout = (const uint8_t*)c.dev_out.p + sl * (slot_out + slot_sz);
        for (uint32_t i = 0; i < cnt; i++) {
            const uint32_t fs = hs[i];
            if (fs < kPngHeaderSize + kPngTrailerSize || fs > cap) return FPNGB_ERR_INTERNAL;
            sizes[first + i] = fs;
            FPNGB_CUDA_OK(cudaMemcpyAsync((uint8_t*)out + (size_t)(first + i) * out_stride, dout + (size_t)i * dstride, fs, cudaMemcpyDeviceToHost, c.copy_out));
        }
        FPNGB_CUDA_OK(cudaEventRecord(ev_out[sl], c.copy_out));
        return 0;
    };

    for (uint32_t k = 0; k < nchunks && result == FPNGB_OK; k++) {
        const int sl = k % kSlots;
        const uint32_t first = k * per_chunk, cnt = (first + per_chunk <= n) ? per_chunk : n - first;
        if (k >= kSlots) { rc = (int)cudaEventSynchronize(ev_out[sl]); if (rc) { result = 1000 + rc; break; } }   // slot's previous files have left the device
        uint8_t* din = (uint8_t*)c.dev_in.p + sl * slot_in;
        uint8_t* dout = (uint8_t*)c.dev_out.p + sl * (slot_out + slot_sz);
        uint32_t* dsz = (uint32_t*)(dout + slot_out);
        const uint8_t* src = (const uint8_t*)pixels + (size_t)first * image_stride;
        cudaError_t e = contiguous ? cudaMemcpyAsync(din, src, cnt * in_bytes, cudaMemcpyHostToDevice, c.copy_in)
                                   : cudaMemcpy2DAsync(din, in_bytes, src, image_stride, in_bytes, cnt, cudaMemcpyHostToDevice, c.copy_in);
        if (e != cudaSuccess) { result = 1000 + (int)e; break; }
        cudaEventRecord(ev_in[sl], c.copy_in);
        cudaStreamWaitEvent(c.stream, ev_in[sl], 0);
        rc = encode_batch_locked(c, din, tight_layout(w, chans, in_bytes), uint8_format(), cnt, w, h, chans, flags, dout, dstride, dsz, c.stream);
        if (rc) { result = rc; break; }
        cudaEventRecord(ev_done[sl], c.stream);
        cudaStreamWaitEvent(c.copy_out, ev_done[sl], 0);
        cudaMemcpyAsync((uint8_t*)c.pin_small.p + sl * slot_sz, dsz, cnt * 4, cudaMemcpyDeviceToHost, c.copy_out);
        cudaEventRecord(ev_sizes[sl], c.copy_out);
        if (k >= 1) { rc = finish(k - 1); if (rc) { result = rc; break; } }
    }
    if (result == FPNGB_OK) result = finish(nchunks - 1);
    cudaStreamSynchronize(c.copy_in); cudaStreamSynchronize(c.stream); cudaStreamSynchronize(c.copy_out);
    if (result == FPNGB_OK) { cudaError_t e = cudaGetLastError(); if (e != cudaSuccess) result = 1000 + (int)e; }
    return result;
}

// Per-kernel device times (ms) averaged over the encode calls since the last read; slots in ProfSlot order:
// hist, huffman, scan, offsets, fused, finish, pack, adler, crc, conversion pre-pass (slot 9: the *_typed calls, the uint8 copy of a
// strided batch bound for the single-pass encoder, the label and reduce pre-passes), colour-type analysis (slot 10:
// FPNGB_ENCODE_REDUCE), LZ77 match kernel (slot 11: FPNGB_LZ77_CHAIN).  A caller asking for 9 slots gets the first nine.  Returns the number
// of calls averaged.
FPNGB_API int fpngb_profile_enable(int on)
{
    std::lock_guard<std::mutex> lk(g_ctx.mu);
    g_profile = on != 0;
    return 0;
}
FPNGB_API int fpngb_profile_read(float* ms, int nslots)
{
    std::lock_guard<std::mutex> lk(g_ctx.mu);
    double sum[kProfSlots] = {0};
    uint64_t first_call = ~0ull, last_call = 0;
    for (ProfSet* ps : g_prof_sets) {
        int last = 0;   // index of the last recorded event
        cudaEventSynchronize(ps->ev[0]);
        for (int i = 0; i < kProfSlots; i++) {
            if (!ps->used[i]) continue;
            float t = 0;
            cudaEventSynchronize(ps->ev[i + 1]);
            // the CRC of a chunk may run on the side stream, overlapped with the next chunk: its own start event brackets it
            // and the conversion pre-pass, which runs before slot 0 opens
            const bool own_start = (i == kProfCrc && ps->crc_side) || i == kProfConvert || i == kProfReduce || i == kProfMatch;
            cudaEvent_t from = i == kProfConvert ? ps->conv_start : i == kProfReduce ? ps->red_start : i == kProfMatch ? ps->ev[kProfHist + 1]
                             : own_start ? ps->crc_start : ps->ev[last];
            if (i == kProfHuff && ps->used[kProfMatch]) from = ps->ev[kProfMatch + 1];
            if (cudaEventElapsedTime(&t, from, ps->ev[i + 1]) == cudaSuccess) sum[i] += t;
            if (!own_start) last = i + 1;
        }
        if (ps->call < first_call) first_call = ps->call;
        if (ps->call > last_call) last_call = ps->call;
        g_prof_free.push_back(ps);
    }
    const int calls = g_prof_sets.empty() ? 0 : (int)(last_call - first_call + 1);
    g_prof_sets.clear();
    for (int i = 0; i < nslots && i < kProfSlots; i++) ms[i] = calls ? (float)(sum[i] / calls) : 0.f;
    return calls;
}

// fpng_crc32 / fpng_adler32 utilities (src/fpng.h:26-31) on host buffers.  Buffers of at least 4 KiB go through the
// device kernels; shorter ones (chunk headers, IHDR) and calls made before fpngb_init() use the host table that the
// container code needs anyway (documented in include/fpng_b200.h).  The *_ex forms report device errors; the plain forms
// keep the reference's signatures and, because 0 is a valid checksum, report a device failure on stderr before returning 0.
int fpngb_crc32_ex(const void* data, size_t size, uint32_t prev, uint32_t* out)
{
    if (!out) return FPNGB_ERR_INVALID_ARG;
    *out = prev;
    if (!data || !size) return FPNGB_OK;
    if (!g_ctx.ready || size < 4096 || size > 0xFFFFFF00ull) { *out = host_crc32(data, size, prev); return FPNGB_OK; }
    Context& c = g_ctx;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    // the buffer stands where "IDAT" + zlib stream stands in a file, bytes [54, 54 + size): the stream CRC kernel's message
    const size_t msg = kPngHeaderSize - 4, padded = align_up(msg + size + 4, 16);
    int rc = c.dev_in.reserve(padded + 256); if (rc) return rc;
    ImageState hst{}; hst.zsize = (uint32_t)size - 4;                   // kernel computes L = 58 + zsize = 54 + size
    ImageState* dst = (ImageState*)((uint8_t*)c.dev_in.p + padded);
    FPNGB_CUDA_OK(cudaMemcpyAsync((uint8_t*)c.dev_in.p + msg, data, size, cudaMemcpyHostToDevice, c.stream));
    FPNGB_CUDA_OK(cudaMemcpyAsync(dst, &hst, sizeof hst, cudaMemcpyHostToDevice, c.stream));
    CrcParams cp{};
    cp.out = (uint8_t*)c.dev_in.p; cp.st = dst;
    launch_crc_stream(cp, 1, msg + size + 4, c.stream);
    count_launch(1);
    FPNGB_CUDA_OK(cudaGetLastError());
    uint8_t be[4] = {0, 0, 0, 0};
    FPNGB_CUDA_OK(cudaMemcpyAsync(be, (uint8_t*)c.dev_in.p + msg + size, 4, cudaMemcpyDeviceToHost, c.stream));
    FPNGB_CUDA_OK(cudaStreamSynchronize(c.stream));
    // the kernel starts from a fresh CRC; by linearity crc(prev, M) = crc(0, M) ^ prev * x^(8 |M|)
    *out = (((uint32_t)be[0] << 24) | ((uint32_t)be[1] << 16) | ((uint32_t)be[2] << 8) | be[3]) ^ gf2_mulmod(prev, xpow(8ull * size));
    return FPNGB_OK;
}

int fpngb_adler32_ex(const void* data, size_t size, uint32_t adler, uint32_t* out)
{
    if (!out) return FPNGB_ERR_INVALID_ARG;
    *out = adler;
    uint32_t a = adler & 0xFFFF, b = adler >> 16;
    if (!data || !size) return FPNGB_OK;
    if (!g_ctx.ready || size < 4096) {
        const uint8_t* p = (const uint8_t*)data;
        for (size_t i = 0; i < size; i++) { a = (a + p[i]) % kAdlerMod; b = (b + a) % kAdlerMod; }
        *out = (b << 16) | a;
        return FPNGB_OK;
    }
    Context& c = g_ctx;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    const size_t padded = align_up(size, 256), nchunks = (size + adler_chunk_bytes() - 1) / adler_chunk_bytes();
    int rc = c.dev_in.reserve(padded + nchunks * 8); if (rc) return rc;
    uint2* dpart = (uint2*)((uint8_t*)c.dev_in.p + padded);
    std::vector<uint2> part(nchunks);
    FPNGB_CUDA_OK(cudaMemcpyAsync(c.dev_in.p, data, size, cudaMemcpyHostToDevice, c.stream));
    launch_adler_buffer((const uint8_t*)c.dev_in.p, size, dpart, c.stream);
    count_launch(1);
    FPNGB_CUDA_OK(cudaGetLastError());
    FPNGB_CUDA_OK(cudaMemcpyAsync(part.data(), dpart, nchunks * 8, cudaMemcpyDeviceToHost, c.stream));
    FPNGB_CUDA_OK(cudaStreamSynchronize(c.stream));
    unsigned long long A = a, B = b;
    for (size_t i = 0; i < nchunks; i++) {
        const unsigned long long len = (i + 1 < nchunks) ? adler_chunk_bytes() : size - i * adler_chunk_bytes();
        B = (B + (len % kAdlerMod) * A + part[i].y) % kAdlerMod;
        A = (A + part[i].x) % kAdlerMod;
    }
    *out = (uint32_t)((B << 16) | A);
    return FPNGB_OK;
}

uint32_t fpngb_crc32(const void* data, size_t size, uint32_t prev)
{
    uint32_t v = 0;
    const int rc = fpngb_crc32_ex(data, size, prev, &v);
    if (rc) { fprintf(stderr, "fpng_b200: fpng_crc32 failed on the device (error %d); the returned value is NOT a checksum\n", rc); return 0; }
    return v;
}

uint32_t fpngb_adler32(const void* data, size_t size, uint32_t adler)
{
    uint32_t v = 0;
    const int rc = fpngb_adler32_ex(data, size, adler, &v);
    if (rc) { fprintf(stderr, "fpng_b200: fpng_adler32 failed on the device (error %d); the returned value is NOT a checksum\n", rc); return 0; }
    return v;
}

int fpngb_compact_batch_device(const void* d_files, size_t stride, const uint32_t* d_sizes, uint32_t n, void* d_dst, size_t dst_cap,
                               uint64_t* d_offsets, void* stream)
{
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!d_files || !d_sizes || !d_dst || !d_offsets || n == 0 || n > 65535) return FPNGB_ERR_INVALID_ARG;
    if (stride % 16 || (uintptr_t)d_files % 16 || (uintptr_t)d_dst % 16) return FPNGB_ERR_ALIGNMENT;
    FPNGB_CUDA_OK(cudaSetDevice(g_ctx.device));
    launch_compact((const uint8_t*)d_files, stride, d_sizes, n, (uint8_t*)d_dst, dst_cap, (unsigned long long*)d_offsets, (cudaStream_t)stream);
    count_launch(2);
    FPNGB_CUDA_OK(cudaGetLastError());
    return FPNGB_OK;
}

int fpngb_compact_packed_device(const void* d_base, const uint64_t* d_src_offsets, const uint32_t* d_sizes, uint32_t n, void* d_dst,
                                size_t dst_cap, uint64_t* d_offsets, void* stream)
{
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!d_base || !d_src_offsets || !d_sizes || !d_dst || !d_offsets || n == 0 || n > 65535) return FPNGB_ERR_INVALID_ARG;
    if ((uintptr_t)d_base % 16 || (uintptr_t)d_dst % 16) return FPNGB_ERR_ALIGNMENT;
    FPNGB_CUDA_OK(cudaSetDevice(g_ctx.device));
    launch_compact((const uint8_t*)d_base, 0, d_sizes, n, (uint8_t*)d_dst, dst_cap, (unsigned long long*)d_offsets, (cudaStream_t)stream,
                   (const unsigned long long*)d_src_offsets);
    count_launch(2);
    FPNGB_CUDA_OK(cudaGetLastError());
    return FPNGB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Static-table training (SURVEY section 8f rank 3; reference: fpng_test -t, src/fpng_test.cpp:766-963, and
// create_dynamic_block_prefix, src/fpng.cpp:909-988).  The GPU part is the 288-bin histogram kernel of 2-pass mode.
// ---------------------------------------------------------------------------------------------------------
// Adds, for every image of a device-resident batch, its 16-bit scaled symbol counts to counts[288] -- exactly what the
// reference accumulates in g_huff_counts while encoding with FPNG_ENCODE_SLOWER (fpng.cpp:751-755 after 1092-1094).
int fpngb_train_accumulate_device(const void* d_pixels, size_t image_stride, uint32_t n, uint32_t w, uint32_t h, uint32_t chans,
                                  uint64_t* counts, void* stream)
{
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!d_pixels || !counts || n == 0 || !valid_dims(w, h, chans) || image_stride < (size_t)w * h * chans || n > 65535) return FPNGB_ERR_INVALID_ARG;
    Context& c = g_ctx;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    cudaStream_t s = (cudaStream_t)stream;
    Workspace ws;
    int rc = carve_workspace(c, n, h, w, true, ws); if (rc) return rc;
    rc = c.ws_acquire(s); if (rc) return rc;
    ScanParams sp{};
    sp.pixels = (const uint8_t*)d_pixels; sp.image_stride = image_stride; sp.row_pitch = w * chans; sp.w = w; sp.h = h; sp.books = c.d_static_books; sp.book_stride = 0;
    sp.row_bits = ws.row_bits; sp.row_adler = ws.row_adler; sp.st = ws.st; sp.hist = ws.hist; sp.lane_ofs = ws.lane_ofs; sp.lane_ofs_pitch = ws.lane_ofs_pitch;
    FPNGB_CUDA_OK(cudaMemsetAsync(ws.hist, 0, (size_t)n * 288 * 4, s));
    launch_hist16(sp, n, chans, s);
    count_launch(1);
    std::vector<uint32_t> hh((size_t)n * 288);
    FPNGB_CUDA_OK(cudaMemcpyAsync(hh.data(), ws.hist, hh.size() * 4, cudaMemcpyDeviceToHost, s));
    rc = c.ws_release(s); if (rc) return rc;
    FPNGB_CUDA_OK(cudaStreamSynchronize(s));
    for (uint32_t i = 0; i < n; i++) {
        uint32_t* f = &hh[(size_t)i * 288];
        f[256] = 1;                                                   // fpng.cpp:1092
        uint64_t total = 0;
        for (int k = 0; k < 288; k++) total += f[k];
        for (int k = 0; k < 288; k++) if (f[k]) { uint64_t v = (uint64_t)f[k] * 65535u / total; counts[k] += v < 1 ? 1 : v; }   // fpng.cpp:890
    }
    return FPNGB_OK;
}

// counts[288] -> pre-serialised block header ("prefix": zlib header, BFINAL, BTYPE=2, table description), the bits left
// over after the last whole byte, and the code table.  Same signature/semantics as the reference's
// create_dynamic_block_prefix (fpng.cpp:910).  The table construction runs in the Huffman-build kernel.
int fpngb_create_dynamic_block_prefix(const uint64_t* counts, uint32_t chans, uint8_t* prefix, size_t prefix_cap, size_t* prefix_len,
                                      uint64_t* bit_buf, int* bit_buf_size, uint32_t* codes288, uint8_t* sizes288)
{
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!counts || !prefix || !prefix_len || !bit_buf || !bit_buf_size || (chans != 3 && chans != 4)) return FPNGB_ERR_INVALID_ARG;
    uint32_t freq[288];
    for (int i = 0; i < 288; i++) freq[i] = (uint32_t)counts[i];       // fpng.cpp:933 (the reference stores the unshifted count)
    for (int i = 0; i <= 256; i++) if (!freq[i]) freq[i] = 1;          // every literal / EOB codable (fpng.cpp:943-947)
    for (uint32_t len = chans; len <= 258; len += chans) { uint32_t sym, xb, xv; deflate_len_code(len, sym, xb, xv); if (!freq[sym]) freq[sym] = 1; }
    Context& c = g_ctx;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    int rc = c.dev_in.reserve(288 * 4 + sizeof(CodeBook) + 512); if (rc) return rc;
    uint32_t* d_hist = (uint32_t*)c.dev_in.p;
    CodeBook* d_book = (CodeBook*)((uint8_t*)c.dev_in.p + 2048);
    FPNGB_CUDA_OK(cudaMemcpyAsync(d_hist, freq, sizeof freq, cudaMemcpyHostToDevice, c.stream));
    HuffParams hp{d_hist, d_book, chans, 1u};
    launch_huffman_build(hp, 1, c.stream);
    count_launch(1);
    static CodeBook hb;
    FPNGB_CUDA_OK(cudaMemcpyAsync(&hb, d_book, sizeof hb, cudaMemcpyDeviceToHost, c.stream));
    FPNGB_CUDA_OK(cudaStreamSynchronize(c.stream));
    const size_t nbytes = hb.hdr_bits / 8;
    if (prefix_cap < nbytes) return FPNGB_ERR_BUFFER_TOO_SMALL;
    memcpy(prefix, hb.hdr, nbytes);
    *prefix_len = nbytes;
    *bit_buf_size = (int)(hb.hdr_bits & 7);
    *bit_buf = hb.hdr[nbytes] & ((1u << (hb.hdr_bits & 7)) - 1u);
    // the exported code table covers every symbol with a code (canonical assignment, fpng.cpp:701-708), including
    // length symbols this encoder never emits
    uint16_t codes16[288];
    canonical_codes(hb.sym_size, 288, codes16);
    for (int i = 0; i < 288; i++) {
        if (sizes288) sizes288[i] = hb.sym_size[i];
        if (codes288) codes288[i] = codes16[i];
    }
    return FPNGB_OK;
}

// Install a trained 1-pass table (prefix bytes + leftover bits, as produced above or by the reference's trainer) for
// `chans`; nbytes == 0 restores the built-in table.  Files written with it are ordinary fpng files.
int fpngb_set_static_table(uint32_t chans, const uint8_t* prefix, size_t nbytes, uint32_t bit_buf, uint32_t bit_buf_size)
{
    if (!g_ctx.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (chans != 3 && chans != 4) return FPNGB_ERR_INVALID_ARG;
    Context& c = g_ctx;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    static CodeBook cb;                                                // static: still alive while the async copy runs
    bool ok;
    if (nbytes == 0) ok = chans == 3 ? build_static_book(cb, kStaticHdrRGB, sizeof kStaticHdrRGB, kStaticHdrRGBTail, kStaticHdrRGBTailBits, 3)
                                     : build_static_book(cb, kStaticHdrRGBA, sizeof kStaticHdrRGBA, kStaticHdrRGBATail, kStaticHdrRGBATailBits, 4);
    else {
        if (!prefix || nbytes + 1 > kMaxHdrBytes || bit_buf_size > 7) return FPNGB_ERR_INVALID_ARG;
        ok = build_static_book(cb, prefix, (uint32_t)nbytes, bit_buf, bit_buf_size, chans);
    }
    if (!ok) return FPNGB_ERR_INVALID_ARG;
    FPNGB_CUDA_OK(cudaDeviceSynchronize());                            // no encode may be using the old table
    c.h_static_books[chans == 4 ? 1 : 0] = cb;
    FPNGB_CUDA_OK(cudaMemcpy(c.d_static_books + (chans == 4 ? 1 : 0), &cb, sizeof cb, cudaMemcpyHostToDevice));
    return FPNGB_OK;
}

// Binds the calling thread (and the threads it creates later) to the CPUs of the NUMA node the library's GPU hangs off, so that
// pinned staging buffers allocated afterwards (first touch) and the copy-issuing thread sit next to the GPU's PCIe root port.
// With 8 ranks on a two-socket host this is what keeps H2D/D2H of the *_host entry points from crossing the socket
// interconnect.  Returns the NUMA node (>= 0), or -1 when the topology is not exposed (single node, container without
// sysfs): then nothing is changed.
int fpngb_bind_host_thread_to_device_numa(void)
{
    if (!g_ctx.ready) return -1;
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, g_ctx.device) != cudaSuccess) return -1;
    for (char* q = bus; *q; q++) if (*q >= 'A' && *q <= 'Z') *q = (char)(*q - 'A' + 'a');
    char path[160];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    if (node < 0) return -1;
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r");
    if (!f) return -1;
    char list[4096] = {0};
    const size_t got = fread(list, 1, sizeof list - 1, f);
    fclose(f);
    if (!got) return -1;
    cpu_set_t set; CPU_ZERO(&set);
    cpu_set_t allowed; CPU_ZERO(&allowed);
    if (sched_getaffinity(0, sizeof allowed, &allowed) != 0) return -1;
    int count = 0;
    for (char* tok = strtok(list, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
        int a = 0, b = 0;
        if (sscanf(tok, "%d-%d", &a, &b) == 2) { } else if (sscanf(tok, "%d", &a) == 1) b = a; else continue;
        for (int c = a; c <= b && c < CPU_SETSIZE; c++) if (CPU_ISSET(c, &allowed)) { CPU_SET(c, &set); count++; }
    }
    if (!count) return -1;                                             // the node's CPUs are outside this process's cpuset: leave it alone
    if (sched_setaffinity(0, sizeof set, &set) != 0) return -1;
    return node;
}

void* fpngb_host_alloc(size_t bytes)
{
    void* p = nullptr;
    if (cudaMallocHost(&p, bytes) != cudaSuccess) return nullptr;
    return p;
}
void fpngb_host_free(void* p) { if (p) cudaFreeHost(p); }

}  // extern "C"
