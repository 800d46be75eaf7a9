// fpng_b200/csrc/inflate_kernels.cu -- gather and inflate of the general PNG files (png_walk.cuh) of the any-PNG decodes.
//
// png_gather_kernel: one CTA per file copies the payloads of the file's consecutive IDAT chunks back to back into the workspace, so
//   that the inflate reads one contiguous zlib stream.  With verify on it also checks every IDAT chunk's CRC-32 in parallel: each
//   thread runs the byte-table register over a contiguous slice of "IDAT" + data, advances it over the bytes behind its slice
//   (multiplication by x^(8 m), from a table of x^(8 * 2^k)), and the CTA XOR-reduces the shares (crc_math.cuh's arithmetic).
// png_inflate_kernel: one warp per file.  Deflate block boundaries are only known once the previous block is decoded, so a file is
//   serial across its blocks; inside a block every lane runs the same symbol decode on the same bit buffer (warp-uniform control
//   flow, no shuffles), the input comes through a 512-byte shared window the warp refills with one coalesced load, literals collect
//   one per lane and go out as one store per run, and the warp copies each match: byte j of a match of distance d is
//   out[start - d + (j mod d)], always written before the match starts.  Huffman tables: a 1024-entry (10-bit) primary table per
//   code for every code of at most 10 bits, and the canonical count / sorted-symbol walk (RFC 1951 3.2.2) for the longer ones.
//   Acceptance is zlib's inflate (inflate.c / inftrees.c): over-subscribed codes, incomplete codes (except a lit/len or distance
//   code with one code of length 1, or no distance codes), HLIT > 286, HDIST > 30, a repeat with no previous length or past the
//   end, no end-of-block code, lit/len 286 / 287, distance 30 / 31, a distance before the start of the stream, a stored length
//   whose complement does not match, block type 3, and input ending before the final block does: FAILED_INVALID_IDAT.  So are
//   a bad zlib header, an inflated size other than h * (1 + w*chans) (PngDesc::raw_len for the ext files of FPNGB_PNG_ALL_FORMATS)
//   and a filter byte above 4 (checked here for 8-bit files, by png_unfilter_ext_kernel for ext files).  With verify on the Adler-32 of the
//   inflated bytes (per-lane sums and the closed form of decode_adler_kernel) is checked against the four bytes behind the final
//   block: FPNGB_DECODE_ADLER_MISMATCH when they differ or are missing.
#include "decode.cuh"
#include "crc_math.cuh"
#include "../../include/fpng_b200.h"

namespace fpngb {

// ---- gather -------------------------------------------------------------------------------------------------------------------
struct PngCrcTables { uint32_t byte[256]; uint32_t x8pow[32]; };   // byte table; x^(8 * 2^k) in the reflected form of crc_math.cuh
static constexpr PngCrcTables make_png_crc_tables()
{
    PngCrcTables r{};
    const CrcByteTable b = crc_byte_table();
    for (uint32_t n = 0; n < 256; n++) r.byte[n] = b.t[n];
    r.x8pow[0] = kCrcOne >> 8;                                               // x^8
    for (int k = 1; k < 32; k++) r.x8pow[k] = gf2_mulmod(r.x8pow[k - 1], r.x8pow[k - 1]);
    return r;
}
__constant__ PngCrcTables c_png_crc = make_png_crc_tables();

__device__ __forceinline__ uint32_t png_be32(const uint8_t* p)
{
    return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3];
}
// r advanced over m zero bytes
__device__ __forceinline__ uint32_t crc_shift(uint32_t r, uint32_t m, const uint32_t* pow)
{
    for (int k = 0; m; k++, m >>= 1)
        if (m & 1u) r = gf2_mulmod(r, pow[k]);
    return r;
}

constexpr uint32_t kGatherThreads = 256;
__global__ void __launch_bounds__(kGatherThreads) png_gather_kernel(PngParams p)
{
    __shared__ PngCrcTables s_tab;
    __shared__ uint32_t s_red[kGatherThreads / 32];
    const uint32_t f = blockIdx.x, tid = threadIdx.x;
    const FileDesc fd = p.files[f];
    if (!png_pending(fd.pre_status)) return;                               // the same for the whole CTA
    if (p.verify) {
        for (uint32_t i = tid; i < 256 + 32; i += kGatherThreads) (&s_tab.byte[0])[i] = (&c_png_crc.byte[0])[i];
        __syncthreads();
    }
    const uint8_t* file = p.d_files + fd.base;
    uint8_t* dst = p.z + p.png[f].zofs;
    uint32_t ofs = fd.idat_ofs, pos = 0;
    bool bad = false;
    // the walk checked the framing: a run of IDAT chunks, then another chunk, all inside the file
    while ((unsigned long long)ofs + 12 <= fd.file_size && file[ofs + 4] == 'I' && file[ofs + 5] == 'D' && file[ofs + 6] == 'A' &&
           file[ofs + 7] == 'T') {
        const uint32_t len = png_be32(file + ofs);
        const uint8_t* src = file + ofs + 8;
        for (uint32_t j = tid; j < len; j += kGatherThreads) dst[pos + j] = src[j];
        if (p.verify) {
            const uint8_t* msg = file + ofs + 4;                             // "IDAT" + data
            const uint32_t m = len + 4, seg = (m + kGatherThreads - 1) / kGatherThreads;
            const uint32_t b0 = min(m, tid * seg), b1 = min(m, b0 + seg);
            uint32_t r = 0;
            for (uint32_t b = b0; b < b1; b++) r = s_tab.byte[(r ^ msg[b]) & 0xFFu] ^ (r >> 8);
            r = crc_shift(r, m - b1, s_tab.x8pow);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) r ^= __shfl_xor_sync(0xFFFFFFFFu, r, o);
            if ((tid & 31u) == 0) s_red[tid >> 5] = r;
            __syncthreads();
            if (tid == 0) {
                uint32_t l = 0;
                for (uint32_t k = 0; k < kGatherThreads / 32; k++) l ^= s_red[k];
                const uint32_t crc = ~(l ^ crc_shift(0xFFFFFFFFu, m, s_tab.x8pow));
                if (crc != png_be32(src + len)) bad = true;
            }
            __syncthreads();
        }
        pos += len;
        ofs += 12 + len;
    }
    if (tid == 0 && bad) p.png[f].status = FPNGB_DECODE_FAILED_HEADER_CRC32;
}

// ---- inflate ------------------------------------------------------------------------------------------------------------------
constexpr uint32_t kInflateWarps = 4;
constexpr uint32_t kFastBits = 10;
constexpr uint32_t kWinWords = 128;                 // 512-byte input window per warp

struct HuffTable {
    uint16_t fast[1 << kFastBits];                  // sym | len << 9 for the codes of <= kFastBits bits, indexed by the next bits; 0: none
    uint16_t count[16];                             // codes per length
    uint16_t first[16], offs[16];                   // canonical first code and first sorted index per length (scratch of the build)
};
struct InflateSmem {
    uint32_t win[kWinWords];
    HuffTable lit, dist;
    uint16_t lsym[288], dsym[32];                   // symbols sorted by code
    uint8_t lens[288 + 32];
    uint8_t clens[20];
};

__constant__ uint16_t c_len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                                        131, 163, 195, 227, 258};
__constant__ uint8_t c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dist_base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
                                         2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_clen_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// Bit reader over the gathered stream; every lane holds the same state.  Bits past the stream read as 0; past() tells.
struct BitReader {
    const uint32_t* z;                              // the stream, 4-byte aligned
    uint32_t* win;                                  // shared window: bytes [wbase, wbase + 512)
    uint32_t zlen, padded, pos, wbase, bc;          // pos: next byte to load into bb (a multiple of 4)
    unsigned long long bb;

    __device__ __forceinline__ void load_window(uint32_t lane)
    {
        wbase = pos;
        __syncwarp();
#pragma unroll
        for (uint32_t k = 0; k < kWinWords / 32; k++) {
            const uint32_t b = wbase + 4u * (lane + 32u * k);
            win[lane + 32u * k] = b < padded ? z[b >> 2] : 0u;
        }
        __syncwarp();
    }
    __device__ __forceinline__ void need(uint32_t lane)   // at least 32 bits in bb
    {
        if (bc < 32) {
            if (pos - wbase >= 4u * kWinWords) load_window(lane);
            bb |= (unsigned long long)win[(pos - wbase) >> 2] << bc;
            bc += 32; pos += 4;
        }
    }
    __device__ __forceinline__ uint32_t take(uint32_t n)  // n <= bc
    {
        const uint32_t v = (uint32_t)bb & ((1u << n) - 1u);
        bb >>= n; bc -= n;
        return v;
    }
    __device__ __forceinline__ unsigned long long consumed() const { return 8ull * pos - bc; }   // bits
    __device__ __forceinline__ bool past() const { return consumed() > 8ull * zlen; }
};

// Builds table t and its sorted symbols from lens[0..n) with zlib's acceptance rule (inftrees.c): over-subscribed never,
// incomplete only when `codes` is false and the longest code has 1 bit; no codes at all is accepted (every decode then fails).
__device__ bool build_table(const uint8_t* lens, uint32_t n, HuffTable& t, uint16_t* sym, bool codes, uint32_t lane)
{
    for (uint32_t i = lane; i < (1u << kFastBits); i += 32) t.fast[i] = 0;
    int ok = 1;
    if (lane == 0) {
        for (int l = 0; l < 16; l++) t.count[l] = 0;
        for (uint32_t s = 0; s < n; s++) t.count[lens[s]]++;
        t.count[0] = 0;
        int left = 1, max = 0;
        for (int l = 1; l < 16; l++) { left = (left << 1) - t.count[l]; if (left < 0) ok = 0; if (t.count[l]) max = l; }
        if (ok && max && left > 0 && (codes || max != 1)) ok = 0;
        uint32_t code = 0, idx = 0;
        for (int l = 1; l < 16; l++) { code = (code + t.count[l - 1]) << 1; t.first[l] = (uint16_t)code; t.offs[l] = (uint16_t)idx; idx += t.count[l]; }
        uint16_t next[16];
        for (int l = 1; l < 16; l++) next[l] = t.offs[l];
        if (ok) for (uint32_t s = 0; s < n; s++) if (lens[s]) sym[next[lens[s]]++] = (uint16_t)s;
    }
    ok = __shfl_sync(0xFFFFFFFFu, ok, 0);
    __syncwarp();
    if (!ok) return false;
    uint32_t total = 0;
    for (int l = 1; l < 16; l++) total += t.count[l];
    for (uint32_t k = lane; k < total; k += 32) {
        const uint32_t s = sym[k], l = lens[s];
        if (l > kFastBits) continue;
        const uint32_t code = t.first[l] + (k - t.offs[l]);
        const uint32_t e = s | (l << 9);
        for (uint32_t j = __brev(code) >> (32 - l); j < (1u << kFastBits); j += 1u << l) t.fast[j] = (uint16_t)e;
    }
    __syncwarp();
    return true;
}

// next symbol of table t (br.bc >= 15), or -1 for a bit pattern that is no code
__device__ __forceinline__ int decode_sym(BitReader& br, const HuffTable& t, const uint16_t* sym)
{
    const uint32_t e = t.fast[(uint32_t)br.bb & ((1u << kFastBits) - 1u)];
    if (e) { br.take(e >> 9); return (int)(e & 511u); }
    int code = 0, first = 0, index = 0;
    unsigned long long b = br.bb;
    for (uint32_t l = 1; l < 16; l++) {                                     // canonical walk, one bit per length
        code |= (int)(b & 1ull); b >>= 1;
        const int count = t.count[l];
        if (code - count < first) { br.take(l); return sym[index + (code - first)]; }
        index += count; first += count; first <<= 1; code <<= 1;
    }
    return -1;
}

__global__ void __launch_bounds__(32 * kInflateWarps) png_inflate_kernel(PngParams p)
{
    __shared__ InflateSmem s_all[kInflateWarps];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t f = blockIdx.x * kInflateWarps + warp;
    if (f >= p.n) return;
    const FileDesc fd = p.files[f];
    if (!png_pending(fd.pre_status)) return;
    const bool ext = fd.pre_status == kPngPendingExt;
    const PngDesc pd = p.png[f];
    if (pd.status) return;                                                  // a bad IDAT CRC (verify)
    InflateSmem& sm = s_all[warp];
    uint8_t* out = p.rows + fd.delta_base;
    const uint32_t stride = fd.w * fd.chans + 1u;
    const unsigned long long N = ext ? pd.raw_len : (unsigned long long)fd.h * stride;
    BitReader br;
    br.z = reinterpret_cast<const uint32_t*>(p.z + pd.zofs); br.win = sm.win;
    br.zlen = pd.zlen; br.padded = (pd.zlen + 3u) & ~3u; br.pos = 0; br.bc = 0; br.bb = 0;
    br.load_window(lane);
    bool err = false;
    unsigned long long o = 0;                                               // output bytes
    br.need(lane);
    {
        const uint32_t cmf = br.take(8), flg = br.take(8);
        if ((cmf & 15u) != 8u || (cmf >> 4) > 7u || ((cmf << 8) | flg) % 31u != 0u || (flg & 0x20u)) err = true;
    }
    uint32_t final = 0;
    uint32_t lit_byte = 0, nrun = 0;                                        // literal run: byte `lane` of the run in lane `lane`
    while (!err && !final) {
        br.need(lane);
        final = br.take(1);
        const uint32_t type = br.take(2);
        if (type == 0) {                                                    // stored: whole bytes from the stream, whole warp
            br.take(br.bc & 7u);
            br.need(lane);
            const uint32_t len = br.take(16), nlen = br.take(16);
            if (len != (~nlen & 0xFFFFu)) { err = true; break; }
            const unsigned long long q = br.consumed() >> 3;               // byte-aligned
            if (o + len > N || q + len > br.zlen) { err = true; break; }
            const uint8_t* src = reinterpret_cast<const uint8_t*>(br.z) + q;
            for (uint32_t j = lane; j < len; j += 32) out[o + j] = src[j];
            o += len;
            const uint32_t e = (uint32_t)(q + len);
            br.bb = 0; br.bc = 0; br.pos = e & ~3u;
            if (br.pos - br.wbase >= 4u * kWinWords || br.pos < br.wbase) br.load_window(lane);
            br.need(lane);
            br.take(8u * (e & 3u));
            continue;
        }
        if (type == 3) { err = true; break; }
        if (type == 1) {                                                    // fixed codes (RFC 1951 3.2.6), distance 30 / 31 included
            for (uint32_t s = lane; s < 288 + 32; s += 32)
                sm.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
            __syncwarp();
            build_table(sm.lens, 288, sm.lit, sm.lsym, false, lane);
            build_table(sm.lens + 288, 32, sm.dist, sm.dsym, false, lane);
        } else {                                                            // dynamic
            br.need(lane);
            const uint32_t hlit = br.take(5) + 257, hdist = br.take(5) + 1, hclen = br.take(4) + 4;
            if (hlit > 286 || hdist > 30) { err = true; break; }
            for (uint32_t k = 0; k < 19; k++) {
                if (br.bc < 3) br.need(lane);
                const uint32_t v = k < hclen ? br.take(3) : 0u;
                if (lane == 0) sm.clens[c_clen_order[k]] = (uint8_t)v;
            }
            __syncwarp();
            if (!build_table(sm.clens, 19, sm.lit, sm.lsym, true, lane)) { err = true; break; }
            uint32_t k = 0;
            while (k < hlit + hdist) {
                br.need(lane);
                const int s = decode_sym(br, sm.lit, sm.lsym);
                if (s < 0) { err = true; break; }
                if (s < 16) { if (lane == 0) sm.lens[k] = (uint8_t)s; k++; continue; }
                uint32_t rep, v = 0;
                if (s == 16) {
                    if (k == 0) { err = true; break; }
                    __syncwarp();
                    v = sm.lens[k - 1];
                    rep = 3 + br.take(2);
                } else if (s == 17) rep = 3 + br.take(3);
                else rep = 11 + br.take(7);
                if (k + rep > hlit + hdist) { err = true; break; }
                for (uint32_t j = lane; j < rep; j += 32) sm.lens[k + j] = (uint8_t)v;
                k += rep;
            }
            if (err) break;
            __syncwarp();
            // lit/len lengths at [0, hlit), distance lengths at [hlit, hlit + hdist): move the distances to 288
            uint8_t dl = 0;
            if (lane < hdist) dl = sm.lens[hlit + lane];
            __syncwarp();
            for (uint32_t s = hlit + lane; s < 288; s += 32) sm.lens[s] = 0;
            __syncwarp();
            sm.lens[288 + lane] = lane < hdist ? dl : 0;
            __syncwarp();
            if (sm.lens[256] == 0) { err = true; break; }
            if (!build_table(sm.lens, 288, sm.lit, sm.lsym, false, lane)) { err = true; break; }
            if (!build_table(sm.lens + 288, 32, sm.dist, sm.dsym, false, lane)) { err = true; break; }
        }
        // the symbols of a Huffman block
        for (;;) {
            br.need(lane);
            if (br.pos > br.padded + 8u) { err = true; break; }             // far past the stream: stop (past() decides below)
            const int s = decode_sym(br, sm.lit, sm.lsym);
            if (s < 0) { err = true; break; }
            if (s < 256) {
                if (o + nrun >= N) { err = true; break; }
                if (lane == nrun) lit_byte = (uint32_t)s;
                if (++nrun == 32) { out[o + lane] = (uint8_t)lit_byte; o += 32; nrun = 0; }
                continue;
            }
            if (nrun) { if (lane < nrun) out[o + lane] = (uint8_t)lit_byte; o += nrun; nrun = 0; }
            if (s == 256) break;
            if (s > 285) { err = true; break; }
            const uint32_t li = (uint32_t)s - 257u;
            const uint32_t len = c_len_base[li] + br.take(c_len_extra[li]);
            br.need(lane);
            const int ds = decode_sym(br, sm.dist, sm.dsym);
            if (ds < 0 || ds > 29) { err = true; break; }
            const uint32_t d = c_dist_base[ds] + br.take(c_dist_extra[ds]);
            if (d > o || o + len > N) { err = true; break; }
            __syncwarp();                                                   // every earlier byte is visible to the warp
            uint8_t* dst = out + o;
            const uint8_t* src = dst - d;
            if (d >= len) { if (lane < len) dst[lane] = src[lane]; for (uint32_t j = lane + 32; j < len; j += 32) dst[j] = src[j]; }
            else for (uint32_t j = lane; j < len; j += 32) dst[j] = src[j % d];
            o += len;
        }
    }
    if (!err && (o != N || br.past())) err = true;
    __syncwarp();
    if (!err && !ext) {                                                     // filter bytes (ext files: png_unfilter_ext_kernel)
        bool bad = false;
        for (uint32_t y = lane; y < fd.h; y += 32) bad |= out[(size_t)y * stride] > 4;
        err = __any_sync(0xFFFFFFFFu, bad);
    }
    uint32_t status = err ? (uint32_t)FPNGB_DECODE_FAILED_INVALID_IDAT : 0u;
    if (!err && p.verify) {
        const unsigned long long q = (br.consumed() + 7) >> 3;             // the Adler-32 follows the final block, byte-aligned
        bool ok = q + 4 <= pd.zlen;
        if (ok) {
            const unsigned long long per = (N + 31) / 32, b0 = min(N, per * lane), b1 = min(N, b0 + per);
            unsigned long long s1 = 0, s2 = 0;
            uint32_t im = (uint32_t)(b0 % kAdlerMod);
            for (unsigned long long i = b0; i < b1; i++) {
                const uint32_t x = out[i];
                s1 += x; s2 += (unsigned long long)im * x;
                if (++im == kAdlerMod) im = 0;
            }
            s1 %= kAdlerMod; s2 %= kAdlerMod;
#pragma unroll
            for (int k = 16; k > 0; k >>= 1) { s1 += __shfl_xor_sync(0xFFFFFFFFu, s1, k); s2 += __shfl_xor_sync(0xFFFFFFFFu, s2, k); }
            s1 %= kAdlerMod; s2 %= kAdlerMod;
            const unsigned long long n = N % kAdlerMod;
            const uint32_t A = (uint32_t)((1ull + s1) % kAdlerMod);
            const uint32_t B = (uint32_t)((n + n * s1 % kAdlerMod + kAdlerMod - s2) % kAdlerMod);
            const uint8_t* t = p.z + pd.zofs + q;
            ok = ((B << 16) | A) == (((uint32_t)t[0] << 24) | ((uint32_t)t[1] << 16) | ((uint32_t)t[2] << 8) | t[3]);
        }
        if (!ok) status = FPNGB_DECODE_ADLER_MISMATCH;
    }
    if (lane == 0 && status) p.png[f].status = status;
}

void launch_png_inflate(const PngParams& p, cudaStream_t s)
{
    png_gather_kernel<<<p.n, kGatherThreads, 0, s>>>(p);
    png_inflate_kernel<<<(p.n + kInflateWarps - 1) / kInflateWarps, 32 * kInflateWarps, 0, s>>>(p);
}

}  // namespace fpngb
