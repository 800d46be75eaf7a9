/*
 * oracle/png_encode_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * A plain-C, single-threaded restatement of the file format fpngb_encode_png_ragged_device writes for the images fpng does not
 * encode (gray8, gray+alpha 8, and 16-bit gray, gray+alpha, RGB and RGBA; include/fpng_b200.h and DESIGN §4.6).  It is written
 * from the format rules, not from the kernels: every row is filtered four ways plus "none", the row with the smallest sum of
 * min(b, 256 - b) wins, runs of equal filtered pixels become matches at distance B, and one dynamic block is coded with fpng's
 * 2-pass Huffman construction.
 *
 * It is compiled as one translation unit with fpng_oracle.c (liboracle.so) so that it shares that file's Huffman helpers
 * (scale_freq, huff_from_counts), bit writer, Deflate length table and checksums.
 */
#include "fpng_oracle.c"

#include <stdio.h>

/* The Deflate distance code of distance B (RFC 1951 3.2.5) and its extra bits: 1 -> 0, 2 -> 1, 4 -> 3, 6 -> 4 (+1), 8 -> 5 (+1). */
static void dist_code(uint32_t B, uint32_t* sym, uint32_t* xb, uint32_t* xv)
{
    static const uint16_t base[8] = { 1, 2, 3, 4, 5, 7, 9, 13 };
    static const uint8_t extra[8] = { 0, 0, 0, 0, 1, 1, 2, 2 };
    uint32_t s = 0;
    while (s + 1 < 8 && base[s + 1] <= B) s++;
    *sym = s; *xb = extra[s]; *xv = B - base[s];
}

static uint32_t paeth(uint32_t a, uint32_t b, uint32_t c)
{
    const int p = (int)a + (int)b - (int)c;
    const int pa = abs(p - (int)a), pb = abs(p - (int)b), pc = abs(p - (int)c);
    if (pa <= pb && pa <= pc) return a;
    return pb <= pc ? b : c;
}

/* Filter `type` applied to row `cur` (n bytes) with the row above `up` (zeros above row 0), distance B. */
static void filter_row(int type, const uint8_t* cur, const uint8_t* up, size_t n, uint32_t B, uint8_t* out)
{
    for (size_t i = 0; i < n; i++) {
        const uint32_t x = cur[i], a = i >= B ? cur[i - B] : 0, b = up[i], c = i >= B ? up[i - B] : 0;
        uint32_t pred = 0;
        switch (type) {
        case 1: pred = a; break;
        case 2: pred = b; break;
        case 3: pred = (a + b) >> 1; break;
        case 4: pred = paeth(a, b, c); break;
        default: break;
        }
        out[i] = (uint8_t)(x - pred);
    }
}

typedef struct { uint8_t size[288]; uint16_t code[288]; uint8_t hdr[400]; uint32_t hdr_bits; uint32_t dsym, dxb, dxv; } pngbook;

/* fpng's 2-pass construction with the distance table {d(B): 1 bit, d(B) + 1: 1 bit} and HDIST = d(B) + 2 codes. */
static void png_book(const uint32_t* freq /*288, [256] == 1*/, uint32_t B, pngbook* pb)
{
    uint16_t cnt0[288], cnt2[19] = { 0 };
    memset(pb, 0, sizeof *pb);
    dist_code(B, &pb->dsym, &pb->dxb, &pb->dxv);
    scale_freq(freq, 288, cnt0);
    cnt0[256] = 1;
    huff_from_counts(cnt0, 288, 12, pb->size, pb->code);
    int nlit = 286;
    const int ndist = (int)pb->dsym + 2;
    while (nlit > 257 && !pb->size[nlit - 1]) nlit--;
    uint8_t seq[288 + 32], packed[2 * (288 + 32)];
    memcpy(seq, pb->size, (size_t)nlit);
    for (int i = 0; i < ndist; i++) seq[nlit + i] = (uint32_t)i >= pb->dsym ? 1 : 0;
    const int total = nlit + ndist;
    int np = 0;
    uint32_t zrun = 0, rrun = 0;
    uint8_t prev = 0xFF;
#define FLUSH_REP() do { if (rrun) { if (rrun < 3) { cnt2[prev] = (uint16_t)(cnt2[prev] + rrun); while (rrun--) packed[np++] = prev; } \
        else { cnt2[16]++; packed[np++] = 16; packed[np++] = (uint8_t)(rrun - 3); } rrun = 0; } } while (0)
#define FLUSH_ZERO() do { if (zrun) { if (zrun < 3) { cnt2[0] = (uint16_t)(cnt2[0] + zrun); while (zrun--) packed[np++] = 0; } \
        else if (zrun <= 10) { cnt2[17]++; packed[np++] = 17; packed[np++] = (uint8_t)(zrun - 3); } \
        else { cnt2[18]++; packed[np++] = 18; packed[np++] = (uint8_t)(zrun - 11); } zrun = 0; } } while (0)
    for (int i = 0; i < total; i++) {
        const uint8_t cs = seq[i];
        if (!cs) { FLUSH_REP(); if (++zrun == 138) FLUSH_ZERO(); }
        else {
            FLUSH_ZERO();
            if (cs != prev) { FLUSH_REP(); cnt2[cs]++; packed[np++] = cs; }
            else if (++rrun == 6) FLUSH_REP();
        }
        prev = cs;
    }
    if (rrun) FLUSH_REP(); else FLUSH_ZERO();
#undef FLUSH_REP
#undef FLUSH_ZERO
    uint8_t size2[19]; uint16_t code2[19];
    huff_from_counts(cnt2, 19, 7, size2, code2);
    static const uint8_t order[19] = { 16,17,18,0,8,7,9,6,10,5,11,4,12,3,13,2,14,1,15 };
    bitwr bw = { pb->hdr, 0 };
    wr_bits(&bw, 0x78, 8); wr_bits(&bw, 0x01, 8); wr_bits(&bw, 1, 1); wr_bits(&bw, 2, 2);
    wr_bits(&bw, (uint32_t)(nlit - 257), 5);
    wr_bits(&bw, (uint32_t)(ndist - 1), 5);
    int nbl = 18;
    while (nbl >= 0 && !size2[order[nbl]]) nbl--;
    nbl = nbl + 1 < 4 ? 4 : nbl + 1;
    wr_bits(&bw, (uint32_t)(nbl - 4), 4);
    for (int i = 0; i < nbl; i++) wr_bits(&bw, size2[order[i]], 3);
    for (int i = 0; i < np;) {
        const uint8_t c = packed[i++];
        wr_bits(&bw, code2[c], size2[c]);
        if (c >= 16) wr_bits(&bw, packed[i++], c == 16 ? 2 : (c == 17 ? 3 : 7));
    }
    pb->hdr_bits = (uint32_t)bw.nbits;
}

/* Tokens of one filtered row (filter byte first): a literal byte (len 0, v the byte) or a match of len bytes at distance B. */
typedef struct { uint16_t len; uint8_t v; } ptoken;

static size_t png_tokenise(const uint8_t* frow /*1 + w*B*/, uint32_t w, uint32_t B, ptoken* out)
{
    const uint32_t M = 258 / B, minr = (3 + B - 1) / B;
    const uint8_t* px = frow + 1;
    size_t n = 0;
    out[n].len = 0; out[n].v = frow[0]; n++;
    uint32_t x = 0;
    while (x < w) {
        if (x > 0 && !memcmp(px + (size_t)x * B, px + (size_t)(x - 1) * B, B)) {
            uint32_t e = x;
            while (e < w && !memcmp(px + (size_t)e * B, px + (size_t)(e - 1) * B, B)) e++;
            uint32_t r = e - x;
            while (r >= minr) {
                const uint32_t t = r < M ? r : M;
                out[n].len = (uint16_t)(t * B); out[n].v = 0; n++;
                r -= t; x += t;
            }
            for (; r; r--, x++) for (uint32_t j = 0; j < B; j++) { out[n].len = 0; out[n].v = px[(size_t)x * B + j]; n++; }
            continue;
        }
        for (uint32_t j = 0; j < B; j++) { out[n].len = 0; out[n].v = px[(size_t)x * B + j]; n++; }
        x++;
    }
    return n;
}

static void be32w(uint8_t* p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }

/* Encodes one image: pixels are tight HWC rows of chans samples, uint8 (depth 8) or native-endian uint16 (depth 16).  Returns
 * the file size, or 0 when the arguments are invalid or cap is too small.  filters_out (h bytes, optional) receives each row's
 * filter type as written (all 0 for a stored file). */
ORACLE_API size_t oracle_png_encode(const void* pixels, uint32_t w, uint32_t h, uint32_t chans, uint32_t depth, uint32_t flags,
                                    uint8_t* out, size_t cap, uint8_t* filters_out)
{
    if (!pixels || !out || !w || !h || chans < 1 || chans > 4 || (depth != 8 && depth != 16) || (flags & ~3u)) return 0;
    if (!g_len_sym[3]) len_setup();
    const uint32_t es = depth / 8, B = chans * es;
    const size_t R = (size_t)w * B, stride = R + 1, raw = stride * h;
    const size_t nblk = (raw + 65534) / 65535, zstored = 2 + raw + 5 * nblk + 4;
    uint8_t* be = (uint8_t*)malloc(R * h);            /* PNG byte order: 16-bit samples big-endian */
    uint8_t* filt = (uint8_t*)malloc(raw);
    uint8_t* cand = (uint8_t*)malloc(R + 1);
    uint8_t* zero = (uint8_t*)calloc(R + 1, 1);
    ptoken* toks = (ptoken*)malloc(sizeof(ptoken) * (R + 2));
    if (!be || !filt || !cand || !zero || !toks) { free(be); free(filt); free(cand); free(zero); free(toks); return 0; }
    for (size_t i = 0; i < R * h; i += es) {
        if (es == 1) be[i] = ((const uint8_t*)pixels)[i];
        else { const uint16_t v = ((const uint16_t*)pixels)[i / 2]; be[i] = (uint8_t)(v >> 8); be[i + 1] = (uint8_t)v; }
    }
    /* row filter: smallest sum of min(b, 256 - b), ties to the lower type */
    for (uint32_t y = 0; y < h; y++) {
        const uint8_t* cur = be + (size_t)y * R;
        const uint8_t* up = y ? cur - R : zero;
        uint64_t best = ~0ull;
        for (int t = 0; t < 5; t++) {
            filter_row(t, cur, up, R, B, cand);
            uint64_t cost = 0;
            for (size_t i = 0; i < R; i++) cost += cand[i] < 128 ? cand[i] : 256u - cand[i];
            if (cost < best) { best = cost; filt[(size_t)y * stride] = (uint8_t)t; memcpy(filt + (size_t)y * stride + 1, cand, R); }
        }
    }
    /* histogram, code book, compressed size */
    uint32_t freq[288] = { 0 };
    for (uint32_t y = 0; y < h; y++) {
        const size_t n = png_tokenise(filt + (size_t)y * stride, w, B, toks);
        for (size_t i = 0; i < n; i++) freq[toks[i].len ? g_len_sym[toks[i].len] : toks[i].v]++;
    }
    freq[256] = 1;
    pngbook pb;
    png_book(freq, B, &pb);
    const uint32_t dbits = 1 + pb.dxb, dval = pb.dxv << 1;      /* distance code d(B) is the 1-bit code 0 */
    uint64_t bits = pb.hdr_bits;
    for (int s = 0; s < 288; s++) if (freq[s] && s != 256) bits += (uint64_t)freq[s] * pb.size[s];
    for (uint32_t y = 0; y < h; y++) {                          /* extra bits and distance bits of the matches */
        const size_t n = png_tokenise(filt + (size_t)y * stride, w, B, toks);
        for (size_t i = 0; i < n; i++) if (toks[i].len) bits += g_len_xb[toks[i].len] + dbits;
    }
    bits += pb.size[256];
    const size_t zcomp = (size_t)((bits + 7) / 8) + 4;
    const int stored = (flags & FLAG_FORCE_UNCOMPRESSED) || zcomp > zstored;
    const size_t zlen = stored ? zstored : zcomp;
    const size_t fsize = 41 + zlen + 16;
    size_t result = 0;
    if (fsize <= cap) {
        memset(out, 0, fsize);
        static const uint8_t sig[8] = { 0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A };
        static const uint8_t ctype[5] = { 0, 0, 4, 2, 6 };
        memcpy(out, sig, 8);
        be32w(out + 8, 13); memcpy(out + 12, "IHDR", 4); be32w(out + 16, w); be32w(out + 20, h);
        out[24] = (uint8_t)depth; out[25] = ctype[chans]; out[26] = 0; out[27] = 0; out[28] = 0;
        be32w(out + 29, oracle_crc32(out + 12, 17, 0));
        be32w(out + 33, (uint32_t)zlen); memcpy(out + 37, "IDAT", 4);
        uint8_t* z = out + 41;
        if (stored) {                                           /* filter 0 on every row, fpng's stored-block layout */
            for (uint32_t y = 0; y < h; y++) { filt[(size_t)y * stride] = 0; memcpy(filt + (size_t)y * stride + 1, be + (size_t)y * R, R); }
            stored_stream(filt, raw, z);
        } else {
            bitwr bw = { z, 0 };
            memcpy(z, pb.hdr, (pb.hdr_bits + 7) / 8);
            bw.nbits = pb.hdr_bits;
            for (uint32_t y = 0; y < h; y++) {
                const size_t n = png_tokenise(filt + (size_t)y * stride, w, B, toks);
                for (size_t i = 0; i < n; i++) {
                    if (!toks[i].len) { wr_bits(&bw, pb.code[toks[i].v], pb.size[toks[i].v]); continue; }
                    const uint32_t L = toks[i].len, s = g_len_sym[L];
                    wr_bits(&bw, pb.code[s], pb.size[s]);
                    wr_bits(&bw, g_len_xv[L], g_len_xb[L]);
                    wr_bits(&bw, dval, (int)dbits);
                }
            }
            wr_bits(&bw, pb.code[256], pb.size[256]);
            if ((bw.nbits + 7) / 8 + 4 != zcomp) { fprintf(stderr, "png oracle: size mismatch\n"); abort(); }
            be32w(z + zcomp - 4, oracle_adler32(filt, raw, 1));
        }
        be32w(out + 41 + zlen, oracle_crc32(out + 37, 4 + zlen, 0));
        static const uint8_t iend[12] = { 0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82 };
        memcpy(out + 45 + zlen, iend, 12);
        if (filters_out) for (uint32_t y = 0; y < h; y++) filters_out[y] = filt[(size_t)y * stride];
        result = fsize;
    }
    free(be); free(filt); free(cand); free(zero); free(toks);
    return result;
}
