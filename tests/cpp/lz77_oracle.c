/*
 * tests/cpp/lz77_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * A plain-C, single-threaded restatement of the LZ77 mode of the PNG encode (FPNGB_LZ77_CHAIN; include/fpng_b200.h "LZ77",
 * DESIGN §4.6 "LZ77"), written from the rule, not from the kernels: the rows are filtered as the other PNG files are, the hash
 * chains are built over the whole filtered stream S in stream order, each 16384-byte segment is parsed greedily on its own, and
 * one dynamic block is coded with fpng's 2-pass Huffman construction for both the literal/length and the distance code.
 *
 * It is one translation unit with oracle/png_encode_oracle.c (and through it oracle/fpng_oracle.c) for the row filters, the
 * Huffman helpers, the bit writer, the stored-block writer and the checksums.
 */
#include "../../oracle/png_encode_oracle.c"

#define LZ_SEG 16384u
#define LZ_WIN 32768u

static uint32_t lz_hash(const uint8_t* s, size_t p)
{
    return (((uint32_t)s[p] << 16 | (uint32_t)s[p + 1] << 8 | (uint32_t)s[p + 2]) * 0x9E3779B1u) >> 17;
}

static void lz_dist_code(uint32_t d, uint32_t* sym, uint32_t* xb, uint32_t* xv)
{
    static const uint16_t base[30] = { 1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537,
                                       2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577 };
    uint32_t s = 0;
    while (s + 1 < 30 && base[s + 1] <= d) s++;
    *sym = s; *xb = s < 4 ? 0 : (s - 2) / 2; *xv = d - base[s];
}

/* The greedy parse of S (n bytes) under chain depth K, one token per call of lz_next.  The chains are built in stream order as the
 * parse goes: every position q < p with q + 3 <= n is inserted before the search at p, newest at the head of its hash.  A chain is
 * walked only to distance 32768, so a ring of 65536 links is enough: the walk never follows a link older than that. */
typedef struct {
    const uint8_t* S; size_t n, row; uint32_t K;
    size_t p, end, ins;
    int64_t head[1 << 15], prev[1 << 16];
    uint64_t stats[4];                   /* matches crossing a row, largest distance, 258-byte matches, matches cut at a segment end */
} lzparse;

static void lz_begin(lzparse* z, const uint8_t* S, size_t n, uint32_t K, size_t row)
{
    memset(z, 0, sizeof *z);
    z->S = S; z->n = n; z->K = K; z->row = row;
    z->end = n < LZ_SEG ? n : LZ_SEG;
    for (uint32_t i = 0; i < (1u << 15); i++) z->head[i] = -1;
}

/* the next token: returns 0 at the end of S; *len 0 is the literal *v, else a match of *len bytes at distance *dist */
static int lz_next(lzparse* z, uint32_t* len, uint32_t* dist, uint32_t* v)
{
    const uint8_t* S = z->S;
    if (z->p >= z->n) return 0;
    if (z->p >= z->end) z->end = z->end + LZ_SEG < z->n ? z->end + LZ_SEG : z->n;
    const size_t p = z->p, end = z->end;
    for (; z->ins < p && z->ins + 3 <= z->n; z->ins++) {
        const uint32_t h = lz_hash(S, z->ins);
        z->prev[z->ins & 0xFFFF] = z->head[h]; z->head[h] = (int64_t)z->ins;
    }
    uint32_t bl = 0, bd = 0;
    if (p + 3 <= end) {
        const uint32_t maxl = end - p < 258 ? (uint32_t)(end - p) : 258;
        int64_t q = z->head[lz_hash(S, p)];
        for (uint32_t k = 0; k < z->K && q >= 0; k++) {
            if (p - (size_t)q > LZ_WIN) break;
            uint32_t l = 0;
            while (l < maxl && S[q + l] == S[p + l]) l++;
            if (l > bl) { bl = l; bd = (uint32_t)(p - (size_t)q); if (l == maxl) break; }
            q = z->prev[q & 0xFFFF];
        }
    }
    if (bl >= 3) {
        if (p / z->row != (p + bl - 1) / z->row) z->stats[0]++;
        if (bd > z->stats[1]) z->stats[1] = bd;
        if (bl == 258) z->stats[2]++;
        if (p + bl == end && bl < 258 && end < z->n && S[p - bd + bl] == S[p + bl]) z->stats[3]++;
        *len = bl; *dist = bd; *v = 0;
        z->p += bl;
    } else {
        *len = 0; *dist = 0; *v = S[p];
        z->p++;
    }
    return 1;
}

typedef struct { uint8_t size[288]; uint16_t code[288]; uint8_t dsize[30]; uint16_t dcode[30]; uint8_t hdr[400]; uint32_t hdr_bits; } lzbook;

static void lz_book(const uint32_t* freq /*288, [256] == 1*/, const uint32_t* dfreq /*30*/, lzbook* b)
{
    uint16_t cnt0[288], dc[30], cnt2[19] = { 0 };
    memset(b, 0, sizeof *b);
    scale_freq(freq, 288, cnt0);
    cnt0[256] = 1;
    huff_from_counts(cnt0, 288, 12, b->size, b->code);
    int used = 0, last = 0;
    for (int i = 0; i < 30; i++) if (dfreq[i]) { used++; last = i; }
    if (used >= 2) {
        scale_freq(dfreq, 30, dc);
        huff_from_counts(dc, 30, 12, b->dsize, b->dcode);
    } else {
        const int s = used ? last : 0;
        b->dsize[s] = b->dsize[s ^ 1] = 1;
        b->dcode[s | 1] = 1;
    }
    int nlit = 286, ndist = 30;
    while (nlit > 257 && !b->size[nlit - 1]) nlit--;
    while (!b->dsize[ndist - 1]) ndist--;
    uint8_t seq[288 + 32], packed[2 * (288 + 32)];
    memcpy(seq, b->size, (size_t)nlit);
    memcpy(seq + nlit, b->dsize, (size_t)ndist);
    const int total = nlit + ndist;
    int np = 0;
    uint32_t zrun = 0, rrun = 0;
    uint8_t prevc = 0xFF;
#define FLUSH_REP() do { if (rrun) { if (rrun < 3) { cnt2[prevc] = (uint16_t)(cnt2[prevc] + rrun); while (rrun--) packed[np++] = prevc; } \
        else { cnt2[16]++; packed[np++] = 16; packed[np++] = (uint8_t)(rrun - 3); } rrun = 0; } } while (0)
#define FLUSH_ZERO() do { if (zrun) { if (zrun < 3) { cnt2[0] = (uint16_t)(cnt2[0] + zrun); while (zrun--) packed[np++] = 0; } \
        else if (zrun <= 10) { cnt2[17]++; packed[np++] = 17; packed[np++] = (uint8_t)(zrun - 3); } \
        else { cnt2[18]++; packed[np++] = 18; packed[np++] = (uint8_t)(zrun - 11); } zrun = 0; } } while (0)
    for (int i = 0; i < total; i++) {
        const uint8_t cs = seq[i];
        if (!cs) { FLUSH_REP(); if (++zrun == 138) FLUSH_ZERO(); }
        else {
            FLUSH_ZERO();
            if (cs != prevc) { FLUSH_REP(); cnt2[cs]++; packed[np++] = cs; }
            else if (++rrun == 6) FLUSH_REP();
        }
        prevc = cs;
    }
    if (rrun) FLUSH_REP(); else FLUSH_ZERO();
#undef FLUSH_REP
#undef FLUSH_ZERO
    uint8_t size2[19]; uint16_t code2[19];
    huff_from_counts(cnt2, 19, 7, size2, code2);
    static const uint8_t order[19] = { 16,17,18,0,8,7,9,6,10,5,11,4,12,3,13,2,14,1,15 };
    bitwr bw = { b->hdr, 0 };
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
    b->hdr_bits = (uint32_t)bw.nbits;
}

/* Encodes one image given as h rows of R bytes in PNG byte order (16-bit samples big-endian, a label map's packed rows), filtered
 * at distance B, behind the L-byte container header hdr (its IDAT length is patched here).  flags: FPNGB_FORCE_UNCOMPRESSED (2)
 * or 0; K: the chain depth.  Returns the file size, or 0 when cap is too small.  info (optional, 8 entries): N, the token count,
 * the distance symbols used, stored (0 / 1), zcomp, zstored, then two of the parse's stats (rows crossed, largest distance);
 * stats (optional, 4 entries): the parse's stats (lzparse). */
ORACLE_API size_t lz77_encode(const uint8_t* rows, uint32_t R, uint32_t h, uint32_t B, const uint8_t* hdr, uint32_t L,
                              uint32_t flags, uint32_t K, uint8_t* out, size_t cap, uint64_t* info, uint64_t* stats)
{
    if (!g_len_sym[3]) len_setup();
    const size_t stride = (size_t)R + 1, n = stride * h;
    const size_t nblk = (n + 65534) / 65535, zstored = 2 + n + 5 * nblk + 4;
    uint8_t* S = (uint8_t*)malloc(n);
    uint8_t* cand = (uint8_t*)malloc(stride);
    uint8_t* zero = (uint8_t*)calloc(stride, 1);
    lzparse* z = (lzparse*)malloc(sizeof(lzparse));
    uint64_t st[4] = { 0, 0, 0, 0 }, ntok = 0, extra = 0;
    for (uint32_t y = 0; y < h; y++) {
        const uint8_t* cur = rows + (size_t)y * R;
        const uint8_t* up = y ? cur - R : zero;
        uint64_t best = ~0ull;
        for (int ty = 0; ty < 5; ty++) {
            filter_row(ty, cur, up, R, B, cand);
            uint64_t cost = 0;
            for (size_t i = 0; i < R; i++) cost += cand[i] < 128 ? cand[i] : 256u - cand[i];
            if (cost < best) { best = cost; S[(size_t)y * stride] = (uint8_t)ty; memcpy(S + (size_t)y * stride + 1, cand, R); }
        }
    }
    /* pass 1: histograms and the extra bits, which the code book does not change */
    uint32_t freq[288] = { 0 }, dfreq[30] = { 0 };
    uint32_t len, dist, v, s_, xb, xv;
    lz_begin(z, S, n, K, stride);
    while (lz_next(z, &len, &dist, &v)) {
        ntok++;
        if (!len) { freq[v]++; continue; }
        freq[g_len_sym[len]]++;
        lz_dist_code(dist, &s_, &xb, &xv); dfreq[s_]++;
        extra += g_len_xb[len] + xb;
    }
    memcpy(st, z->stats, sizeof st);
    freq[256] = 1;
    lzbook bk;
    lz_book(freq, dfreq, &bk);
    uint64_t bits = bk.hdr_bits + extra;
    for (int i = 0; i < 288; i++) if (i != 256) bits += (uint64_t)freq[i] * bk.size[i];
    bits += bk.size[256];
    for (int i = 0; i < 30; i++) bits += (uint64_t)dfreq[i] * bk.dsize[i];
    const size_t zcomp = (size_t)((bits + 7) / 8) + 4;
    const int stored = (flags & FLAG_FORCE_UNCOMPRESSED) || zcomp > zstored;
    const size_t zlen = stored ? zstored : zcomp;
    const size_t fsize = L + zlen + 16;
    if (info) {
        uint32_t dused = 0;
        for (int i = 0; i < 30; i++) dused += dfreq[i] != 0;
        info[0] = n; info[1] = ntok; info[2] = dused; info[3] = (uint64_t)stored; info[4] = zcomp; info[5] = zstored;
        info[6] = st[0]; info[7] = st[1];
    }
    if (stats) memcpy(stats, st, sizeof st);
    size_t result = 0;
    if (out && fsize <= cap) {
        memset(out, 0, fsize);
        memcpy(out, hdr, L);
        be32w(out + L - 8, (uint32_t)zlen);
        uint8_t* zs = out + L;
        if (stored) {
            for (uint32_t y = 0; y < h; y++) { S[(size_t)y * stride] = 0; memcpy(S + (size_t)y * stride + 1, rows + (size_t)y * R, R); }
            stored_stream(S, n, zs);
        } else {
            bitwr bw = { zs, 0 };
            memcpy(zs, bk.hdr, (bk.hdr_bits + 7) / 8);
            bw.nbits = bk.hdr_bits;
            lz_begin(z, S, n, K, stride);                       /* pass 2: the same parse, written */
            while (lz_next(z, &len, &dist, &v)) {
                if (!len) { wr_bits(&bw, bk.code[v], bk.size[v]); continue; }
                const uint32_t ls = g_len_sym[len];
                wr_bits(&bw, bk.code[ls], bk.size[ls]);
                wr_bits(&bw, g_len_xv[len], g_len_xb[len]);
                lz_dist_code(dist, &s_, &xb, &xv);
                wr_bits(&bw, bk.dcode[s_], bk.dsize[s_]);
                wr_bits(&bw, xv, (int)xb);
            }
            wr_bits(&bw, bk.code[256], bk.size[256]);
            if ((bw.nbits + 7) / 8 + 4 != zcomp) { fprintf(stderr, "lz77 oracle: size mismatch\n"); abort(); }
            be32w(zs + zcomp - 4, oracle_adler32(S, n, 1));
        }
        be32w(out + L + zlen, oracle_crc32(out + L - 4, 4 + zlen, 0));
        static const uint8_t iend[12] = { 0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82 };
        memcpy(out + L + 4 + zlen, iend, 12);
        result = fsize;
    }
    free(S); free(cand); free(zero); free(z);
    return result;
}

/* The parse of a given stream S (n bytes, no filtering) under chain depth K, for tests of the rule itself: token i is a literal
 * (len[i] = 0, dist[i] = the byte) or a match (len[i], dist[i]).  Returns the token count (at most n; cap entries are written). */
ORACLE_API size_t lz77_parse(const uint8_t* S, size_t n, uint32_t K, uint16_t* len, uint16_t* dist, size_t cap)
{
    lzparse* z = (lzparse*)malloc(sizeof(lzparse));
    uint32_t l, d, v;
    size_t nt = 0;
    lz_begin(z, S, n, K, n ? n : 1);
    while (lz_next(z, &l, &d, &v)) {
        if (nt < cap) { len[nt] = (uint16_t)l; dist[nt] = (uint16_t)(l ? d : v); }
        nt++;
    }
    free(z);
    return nt;
}
