// fpng_b200/csrc/huffman_kernels.cu -- per-image length-limited Huffman construction for 2-pass mode
// (FPNG_ENCODE_SLOWER, src/fpng.h:38).  One warp per image; the 288-bin histogram produced by the scan kernel is
// turned into the image's CodeBook (kernel-facing code tables + the serialised dynamic block header):
//
//   adjust_freq32            fpng.cpp:868-907   32-bit counts -> 16-bit counts, max(1, f*65535/total)
//   stable sort by count     fpng.cpp:622-636   (2-pass LSD radix sort there; a parallel stable rank sort here)
//   minimum-redundancy lens  fpng.cpp:639-659   Moffat & Katajainen's in-place algorithm
//   length limiting          fpng.cpp:663-674   Kraft-sum fix-up to 12 (lit/len, dist) or 7 (code-length code)
//   canonical codes          fpng.cpp:701-708   bit-reversed for LSB-first emission
//   block header             fpng.cpp:746-816   HLIT/HDIST/HCLEN, RLE of the code sizes with symbols 16/17/18
//
// The result is bit-identical to the reference's tables for the same histogram, so 2-pass files are byte-exact.
#include "kernels.cuh"

namespace fpngb {

void finish_codebook(CodeBook& cb, const uint8_t* sizes, const uint16_t* codes, uint32_t chans);   // host twin in host_api.cu

struct HuffScratch {
    uint16_t key[288];        // sorted counts -> parent links -> depths -> code lengths
    uint16_t sym[288];        // symbol index, sorted with the keys
    uint16_t cnt[288];        // 16-bit symbol counts
    uint16_t ukey[288];       // compacted (used symbols only), unsorted
    uint16_t usym[288];
    uint16_t code[288];
    uint8_t  size[288];
    uint8_t  seq[288 + 32];
    uint8_t  packed[288 + 32];
    uint32_t hdr_words[kMaxHdrBytes / 4];
    uint32_t n_used;
};

__device__ static uint32_t dev_bitrev(uint32_t v, int n) { return __brev(v) >> (32 - n); }

// lane-parallel stable sort of (ukey, usym)[0..n) into (key, sym) ascending by key
__device__ static void rank_sort(HuffScratch& s, uint32_t n, uint32_t lane)
{
    for (uint32_t i = lane; i < n; i += 32) {
        const uint32_t k = s.ukey[i];
        uint32_t r = 0;
        for (uint32_t j = 0; j < n; j++) {
            const uint32_t kj = s.ukey[j];
            r += (kj < k) || (kj == k && j < i);
        }
        s.key[r] = (uint16_t)k; s.sym[r] = s.usym[i];
    }
    __syncwarp();
}

// Serial part (lane 0): lengths from sorted counts, limited to maxlen; writes s.size[] for `table_len` symbols and
// canonical bit-reversed codes into s.code[].
// ATTRIBUTION: the first block is the in-place minimum-redundancy code-length algorithm of Alistair Moffat and Jyrki Katajainen
// ("In-place calculation of minimum-redundancy codes", 1995; reference implementation by the authors, November 1996), which the
// reference also uses and credits (fpng.cpp:638-659, via miniz); the second block is the Kraft-sum length limiter of miniz /
// fpng.cpp:663-674.  Both are restated here on purpose with the SAME order of operations and tie-breaking: 2-pass files are
// byte-identical to the reference's only if equal counts receive the same lengths.
__device__ static void lengths_and_codes(HuffScratch& s, int n, int table_len, int maxlen)
{
    uint16_t* A = s.key;
    if (n == 1) A[0] = 1;
    else if (n >= 2) {
        A[0] = (uint16_t)(A[0] + A[1]);
        int root = 0, leaf = 2;
        for (int nx = 1; nx < n - 1; nx++) {
            uint16_t wt;
            if (leaf >= n || A[root] < A[leaf]) { wt = A[root]; A[root++] = (uint16_t)nx; } else wt = A[leaf++];
            if (leaf >= n || (root < nx && A[root] < A[leaf])) { wt = (uint16_t)(wt + A[root]); A[root++] = (uint16_t)nx; }
            else wt = (uint16_t)(wt + A[leaf++]);
            A[nx] = wt;
        }
        A[n - 2] = 0;
        for (int nx = n - 3; nx >= 0; nx--) A[nx] = (uint16_t)(A[A[nx]] + 1);
        int avail = 1, used = 0, depth = 0, nx = n - 1;
        root = n - 2;
        while (avail > 0) {
            while (root >= 0 && (int)A[root] == depth) { used++; root--; }
            while (avail > used) { A[nx--] = (uint16_t)depth; avail--; }
            avail = 2 * used; depth++; used = 0;
        }
    }
    int cnt[33];
    for (int i = 0; i <= 32; i++) cnt[i] = 0;
    for (int i = 0; i < n; i++) cnt[A[i]]++;
    if (n > 1) {
        for (int l = maxlen + 1; l <= 32; l++) cnt[maxlen] += cnt[l];
        uint32_t total = 0;
        for (int l = maxlen; l > 0; l--) total += (uint32_t)cnt[l] << (maxlen - l);
        while (total != (1u << maxlen)) {
            cnt[maxlen]--;
            for (int l = maxlen - 1; l > 0; l--) if (cnt[l]) { cnt[l]--; cnt[l + 1] += 2; break; }
            total--;
        }
    }
    for (int i = 0; i < table_len; i++) { s.size[i] = 0; s.code[i] = 0; }
    int j = n;
    for (int l = 1; l <= maxlen; l++) for (int k = cnt[l]; k > 0; k--) s.size[s.sym[--j]] = (uint8_t)l;
    uint32_t next[17];
    next[1] = 0;
    for (int l = 2; l <= maxlen; l++) next[l] = (next[l - 1] + cnt[l - 1]) << 1;
    for (int i = 0; i < table_len; i++) { const int l = s.size[i]; if (l) s.code[i] = (uint16_t)dev_bitrev(next[l]++, l); }
}

struct DevBitWriter {
    uint32_t* words; uint32_t nbits;
    __device__ void put(uint32_t v, uint32_t n)
    {
        const uint32_t w = nbits >> 5, o = nbits & 31;
        words[w] |= v << o;
        if (o + n > 32) words[w + 1] |= v >> (32 - o);
        nbits += n;
    }
};

// RAGGED: the channel count is image blockIdx.x's (p.desc) instead of the call's
// PNG: the books of fpngb_encode_png_ragged_device, where p.desc's chans is B, the bytes per pixel.  The distance table is
//   {d(B): 1 bit, d(B) + 1: 1 bit} with d(B) + 2 codes (d(B) the distance code of distance B; for B = 3, 4 fpng's table), and
//   match[j] holds length symbol 257 + j as code | size << 16 (j < 29) instead of fpng's matches in pixels
// LZ (with PNG): the LZ77 books.  The distance code is built from p.dhist by the same construction, or, with fewer than two
//   distance symbols used, is {s: 1 bit, s ^ 1: 1 bit} for the used symbol s (0 if none); HDIST is its last symbol of nonzero
//   length + 1; match[32 + j] holds distance symbol j as code | size << 16 (j < 30)
template <bool RAGGED = false, bool PNG = false, bool LZ = false>
__global__ void __launch_bounds__(32) huffman_build_kernel(HuffParams p)
{
    __shared__ HuffScratch s;
    __shared__ uint8_t s_size0[288];
    __shared__ uint16_t s_code0[288];
    __shared__ uint8_t s_dsize[LZ ? 30 : 1];
    __shared__ uint16_t s_dcode[LZ ? 30 : 1];
    const uint32_t img = blockIdx.x, lane = threadIdx.x;
    const uint32_t* hist = p.hist + (size_t)img * 288;
    CodeBook* cb = p.books + img;
    const uint32_t chans = RAGGED ? p.desc[img].chans : p.chans;

    // --- 16-bit scaled counts (fpng.cpp:1092-1094 then 868-893, then 757)
    uint32_t part = 0;
    const bool training = p.training != 0;
    for (uint32_t i = lane; i < 288; i += 32) part += (i == 256 && !training) ? 1u : hist[i];
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xFFFFFFFFu, part, o);
    const uint32_t total = part;
    for (uint32_t i = lane; i < 288; i += 32) {
        const uint32_t f = (i == 256 && !training) ? 1u : hist[i];
        uint32_t v = 0;
        if (f) { v = (uint32_t)(((unsigned long long)f * 65535ull) / total); if (v < 1) v = 1; }
        if (i == 256) v = 1;
        s.cnt[i] = (uint16_t)v;
    }
    for (uint32_t i = lane; i < kMaxHdrBytes / 4; i += 32) s.hdr_words[i] = 0;
    __syncwarp();

    // --- literal/length table (limit 12)
    if (lane == 0) {
        uint32_t n = 0;
        for (uint32_t i = 0; i < 288; i++) if (s.cnt[i]) { s.ukey[n] = s.cnt[i]; s.usym[n] = (uint16_t)i; n++; }
        s.n_used = n;
    }
    __syncwarp();
    rank_sort(s, s.n_used, lane);
    if (lane == 0) lengths_and_codes(s, (int)s.n_used, 288, 12);
    __syncwarp();
    for (uint32_t i = lane; i < 288; i += 32) { s_size0[i] = s.size[i]; s_code0[i] = s.code[i]; }
    __syncwarp();

    // --- LZ77 distance table (limit 12), from 16-bit scaled counts
    if constexpr (LZ) {
        if (lane == 0) {
            const uint32_t* dh = p.dhist + (size_t)img * 32;
            uint32_t tot = 0, n = 0;
            for (uint32_t i = 0; i < 30; i++) tot += dh[i];
            for (uint32_t i = 0; i < 30; i++) if (dh[i]) {
                const uint32_t v = (uint32_t)(((unsigned long long)dh[i] * 65535ull) / tot);
                s.ukey[n] = (uint16_t)(v < 1 ? 1 : v); s.usym[n] = (uint16_t)i; n++;
            }
            s.n_used = n;
        }
        __syncwarp();
        const uint32_t n = s.n_used;
        rank_sort(s, n, lane);
        if (lane == 0) {
            if (n >= 2) {
                lengths_and_codes(s, (int)n, 30, 12);
                for (int i = 0; i < 30; i++) { s_dsize[i] = s.size[i]; s_dcode[i] = s.code[i]; }
            } else {
                const uint32_t u = n ? s.usym[0] : 0u;
                for (int i = 0; i < 30; i++) { s_dsize[i] = 0; s_dcode[i] = 0; }
                s_dsize[u] = s_dsize[u ^ 1u] = 1;
                s_dcode[u | 1u] = 1;                        // canonical: the lower symbol gets 0
            }
        }
        __syncwarp();
    }

    // --- header (lane 0): the distance table is always {chans-1: 1 bit, chans: 1 bit} (fpng.cpp:1096-1098)
    if (lane == 0) {
        const int dsym = PNG ? (chans <= 4 ? (int)chans - 1 : (chans <= 6 ? 4 : 5)) : (int)chans - 1;
        int nlit = 286, ndist = dsym + 2;
        while (nlit > 257 && !s_size0[nlit - 1]) nlit--;
        for (int i = 0; i < nlit; i++) s.seq[i] = s_size0[i];
        if constexpr (LZ) {
            ndist = 30;
            while (!s_dsize[ndist - 1]) ndist--;
            for (int i = 0; i < ndist; i++) s.seq[nlit + i] = s_dsize[i];
        } else {
            for (int i = 0; i < ndist; i++) s.seq[nlit + i] = (i == dsym || i == dsym + 1) ? 1 : 0;
        }
        const int totalc = nlit + ndist;
        uint16_t cnt2[19];
        for (int i = 0; i < 19; i++) cnt2[i] = 0;
        int np = 0;
        uint32_t zrun = 0, rrun = 0; uint8_t prev = 0xFF;
        auto flush_rep = [&]() {
            if (!rrun) return;
            if (rrun < 3) { cnt2[prev] = (uint16_t)(cnt2[prev] + rrun); while (rrun--) s.packed[np++] = prev; }
            else { cnt2[16]++; s.packed[np++] = 16; s.packed[np++] = (uint8_t)(rrun - 3); }
            rrun = 0;
        };
        auto flush_zero = [&]() {
            if (!zrun) return;
            if (zrun < 3) { cnt2[0] = (uint16_t)(cnt2[0] + zrun); while (zrun--) s.packed[np++] = 0; }
            else if (zrun <= 10) { cnt2[17]++; s.packed[np++] = 17; s.packed[np++] = (uint8_t)(zrun - 3); }
            else { cnt2[18]++; s.packed[np++] = 18; s.packed[np++] = (uint8_t)(zrun - 11); }
            zrun = 0;
        };
        for (int i = 0; i < totalc; i++) {
            const uint8_t cs = s.seq[i];
            if (!cs) { flush_rep(); if (++zrun == 138) flush_zero(); }
            else {
                flush_zero();
                if (cs != prev) { flush_rep(); cnt2[cs]++; s.packed[np++] = cs; }
                else if (++rrun == 6) flush_rep();
            }
            prev = cs;
        }
        if (rrun) flush_rep(); else flush_zero();

        // code-length code (limit 7): stable insertion sort of <= 19 symbols, then the same length/code routine
        uint32_t n2 = 0;
        for (uint32_t i = 0; i < 19; i++) if (cnt2[i]) {
            uint32_t j = n2++;
            while (j > 0 && s.key[j - 1] > cnt2[i]) { s.key[j] = s.key[j - 1]; s.sym[j] = s.sym[j - 1]; j--; }
            s.key[j] = cnt2[i]; s.sym[j] = (uint16_t)i;
        }
        lengths_and_codes(s, (int)n2, 19, 7);

        static const uint8_t order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
        DevBitWriter bw{s.hdr_words, 0};
        bw.put(0x78, 8); bw.put(0x01, 8); bw.put(1, 1); bw.put(2, 2);
        bw.put((uint32_t)(nlit - 257), 5); bw.put((uint32_t)(ndist - 1), 5);
        int nbl = 18;
        while (nbl >= 0 && !s.size[order[nbl]]) nbl--;
        nbl = nbl + 1 < 4 ? 4 : nbl + 1;
        bw.put((uint32_t)(nbl - 4), 4);
        for (int i = 0; i < nbl; i++) bw.put(s.size[order[i]], 3);
        for (int i = 0; i < np;) {
            const uint8_t c = s.packed[i++];
            bw.put(s.code[c], s.size[c]);
            if (c >= 16) bw.put(s.packed[i++], c == 16 ? 2 : (c == 17 ? 3 : 7));
        }
        cb->hdr_bits = bw.nbits;
        cb->eob = s_code0[256] | ((uint32_t)s_size0[256] << 16);
    }
    __syncwarp();

    // --- kernel-facing tables
    for (uint32_t i = lane; i < kMaxHdrBytes; i += 32) cb->hdr[i] = (uint8_t)(s.hdr_words[i >> 2] >> (8 * (i & 3)));
    for (uint32_t v = lane; v < 256; v += 32) { cb->lit[v] = s_code0[v] | ((uint32_t)s_size0[v] << 16); cb->lit_size[v] = s_size0[v]; }
    for (uint32_t i = lane; i < 288; i += 32) cb->sym_size[i] = s_size0[i];
    if constexpr (PNG) {
        for (uint32_t j = lane; j < 88; j += 32) {
            uint32_t v = j < 29 ? s_code0[257 + j] | ((uint32_t)s_size0[257 + j] << 16) : 0u;
            if (LZ && j >= 32 && j < 62) v = s_dcode[j - 32] | ((uint32_t)s_dsize[j - 32] << 16);
            cb->match[j] = v;
            cb->match_bits[j] = 0;
        }
        return;
    }
    const uint32_t M = max_match_pixels(chans);
    for (uint32_t n = lane; n < 88; n += 32) {
        uint32_t m = 0, tb = 0;
        if (n >= 1 && n <= M) {
            uint32_t sym, xb, xv;
            deflate_len_code(n * chans, sym, xb, xv);
            const uint32_t sz = s_size0[sym];
            tb = sz ? sz + xb + 1 : 0;                      // unused lengths never occur in this image
            m = (s_code0[sym] | (xv << sz)) | (tb << 24);
        }
        cb->match[n] = m; cb->match_bits[n] = (uint8_t)tb;
    }
}

void launch_huffman_build(const HuffParams& p, uint32_t n, cudaStream_t s)
{
    huffman_build_kernel<false><<<n, 32, 0, s>>>(p);
}

void launch_huffman_build_ragged(const HuffParams& p, uint32_t n, cudaStream_t s)
{
    huffman_build_kernel<true><<<n, 32, 0, s>>>(p);
}

void launch_huffman_build_png(const HuffParams& p, uint32_t n, cudaStream_t s)
{
    huffman_build_kernel<true, true><<<n, 32, 0, s>>>(p);
}

void launch_huffman_build_lz(const HuffParams& p, uint32_t n, cudaStream_t s)
{
    huffman_build_kernel<true, true, true><<<n, 32, 0, s>>>(p);
}

}  // namespace fpngb
