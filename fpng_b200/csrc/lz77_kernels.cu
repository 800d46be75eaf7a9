// fpng_b200/csrc/lz77_kernels.cu -- sm_90a kernels of the LZ77 mode of the PNG encode (FPNGB_LZ77_CHAIN, include/fpng_b200.h
// "LZ77", DESIGN §4.6 "LZ77").  The row kernel's kPngFilt mode has written each image's filtered stream S; these kernels turn
// S into the tokens and codes of one dynamic block, one CTA per 16 KiB segment of S:
//
//   lz_match_kernel            the segment's window [max(0, seg - 32768), seg end) in shared memory; the hash chains of the window
//                              in stream order (warp 0); every position's best match over at most K chain entries (all threads);
//                              the greedy parse (warp 0) into 16-bit token units and the image's literal/length and distance
//                              histograms
//   huffman_build_kernel<.., LZ>  per image: the literal/length and distance codes (huffman_kernels.cu)
//   lz_segment_kernel<false>   the segment's code bits
//   png_lz_offsets_kernel      per image: bit offset of each segment, compressed-vs-stored decision, container (png_encode_kernels.cu)
//   lz_segment_kernel<true>    the segment's codes at its bit offset (staged in shared memory, whole words out)
//
// A chain only links positions inside the window, and every position a segment's chain can reach at distance <= 32768 is inside
// it, so each segment's parse is the one the sequential rule gives, whatever the partition into CTAs.
#include "row_walk.cuh"
#include "kernels.cuh"

namespace fpngb {

constexpr int kLzThreads = 512;
constexpr int kLzSegThreads = 256;
constexpr uint32_t kLzMaxWin = kLzWindow + kLzSegment;             // window bytes of one segment
constexpr uint32_t kLzNone = 0xFFFFu;                               // end of a chain (window positions are < 49152)
constexpr uint32_t kLzMaxLen = 258;
// dynamic shared memory of lz_match_kernel: the window | the 2^15 chain heads (u16), then the segment's best lengths and distances
// (u16 each) | the chain links of the window (u16) | the literal/length and distance histograms
constexpr size_t kLzHeadBytes = 2u << 15;
constexpr size_t kLzSmem = kLzMaxWin + kLzHeadBytes + 2 * kLzMaxWin + 4 * (288 + 32);
// a segment codes to at most 14 bits per byte of S (a literal <= 12 bits; a 3-byte match <= 12 + 5 + 12 + 13 bits), plus the
// bit offset inside its first word
constexpr uint32_t kLzStageWords = (14 * kLzSegment + 31) / 32 + 2;

__device__ __forceinline__ uint32_t lz_hash(const uint8_t* s, uint32_t i)
{
    return (((uint32_t)s[i] << 16 | (uint32_t)s[i + 1] << 8 | (uint32_t)s[i + 2]) * 0x9E3779B1u) >> 17;
}

// Deflate distance code of distance d (1..32768), RFC 1951 3.2.5
__device__ __forceinline__ void deflate_dist_code(uint32_t d, uint32_t& sym, uint32_t& xb, uint32_t& xv)
{
    if (d <= 4) { sym = d - 1; xb = 0; xv = 0; return; }
    const uint32_t a = d - 1, lg = 31 - __clz(a);
    xb = lg - 1; sym = 2 * lg + ((a >> (lg - 1)) & 1u); xv = a & ((1u << xb) - 1u);
}

__device__ __forceinline__ unsigned long long lz_stream_bytes(const ImageDesc& d)
{
    return ((unsigned long long)d.w * d.chans + 1ull) * d.h;
}

__global__ void __launch_bounds__(kLzThreads) lz_match_kernel(PngLzParams p)
{
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t* win = smem;
    uint16_t* head = reinterpret_cast<uint16_t*>(smem + kLzMaxWin);
    uint16_t* best_len = head;                                    // after the chains are built
    uint16_t* best_dist = head + kLzSegment;
    uint16_t* prev = reinterpret_cast<uint16_t*>(smem + kLzMaxWin + kLzHeadBytes);
    uint32_t* s_hist = reinterpret_cast<uint32_t*>(smem + kLzMaxWin + kLzHeadBytes + 2 * kLzMaxWin);
    uint32_t* s_dhist = s_hist + 288;

    uint32_t seg;
    const uint32_t img = ragged_locate(p.ragged, blockIdx.x, seg);
    const ImageDesc& d = p.ragged.desc[img];
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    const unsigned long long N = lz_stream_bytes(d), s0 = (unsigned long long)seg * kLzSegment;
    const uint32_t seglen = (uint32_t)min((unsigned long long)kLzSegment, N - s0);
    const unsigned long long ws = s0 > kLzWindow ? s0 - kLzWindow : 0ull;
    const uint32_t off = (uint32_t)(s0 - ws), wlen = off + seglen;
    const uint8_t* S = p.lz_s + d.lz_ofs + ws;                   // 16-byte aligned: lz_ofs and ws are

    for (uint32_t i = tid; i < wlen / 16u; i += blockDim.x)
        reinterpret_cast<uint4*>(win)[i] = __ldg(reinterpret_cast<const uint4*>(S) + i);
    for (uint32_t i = (wlen & ~15u) + tid; i < wlen; i += blockDim.x) win[i] = S[i];
    for (uint32_t i = tid; i < kLzHeadBytes / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(head)[i] = 0xFFFFFFFFu;
    for (uint32_t i = tid; i < 288 + 32; i += blockDim.x) s_hist[i] = 0u;
    __syncthreads();

    // chains in stream order: 32 positions per step; a lane's link is the nearest lower lane of equal hash, else the head
    if (warp == 0) {
        const uint32_t npos = wlen > 2u ? wlen - 2u : 0u;
        for (uint32_t b = 0; b < npos; b += 32) {
            const uint32_t i = b + lane;
            const bool v = i < npos;
            const uint32_t h = v ? lz_hash(win, i) : 0x10000u + lane;
            const uint32_t grp = __match_any_sync(kFullMask, h);
            const uint32_t lower = grp & ((1u << lane) - 1u);
            const uint32_t link = v ? (lower ? b + 31u - __clz(lower) : head[h]) : 0u;
            __syncwarp();
            if (v) {
                prev[i] = (uint16_t)link;
                if ((grp >> lane) == 1u) head[h] = (uint16_t)i;        // the last lane of its hash
            }
            __syncwarp();
        }
    }
    __syncthreads();

    // best match of every position: at most K chain entries, hash collisions included, none farther than 32768; the longest,
    // ties to the nearest; stop at the longest possible
    const uint32_t K = p.chain;
    for (uint32_t j = tid; j < seglen; j += blockDim.x) {
        uint32_t bl = 0, bd = 0;
        if (j + 3u <= seglen) {
            const uint32_t pw = off + j, maxl = min(kLzMaxLen, seglen - j);
            uint32_t q = prev[pw];
            for (uint32_t k = 0; k < K && q != kLzNone; k++) {
                if (pw - q > kLzWindow) break;
                if (win[q + bl] == win[pw + bl]) {                     // a longer match must agree at index bl
                    uint32_t l = 0;
                    while (l < maxl && win[q + l] == win[pw + l]) l++;
                    if (l > bl) { bl = l; bd = pw - q; if (l == maxl) break; }
                }
                q = prev[q];
            }
        }
        best_len[j] = (uint16_t)(bl >= 3u ? bl : 0u);
        best_dist[j] = (uint16_t)bd;
    }
    __syncthreads();

    // greedy parse, 32 positions per step: the literals before the first match, then the match
    if (warp == 0) {
        uint16_t* tok = p.lz_tok + d.lz_ofs + s0;
        uint32_t pos = 0, t = 0;
        while (pos < seglen) {
            const uint32_t j = pos + lane;
            const bool in = j < seglen;
            const uint32_t L = in ? best_len[j] : 0u, D = in ? best_dist[j] : 0u;
            const uint32_t mb = __ballot_sync(kFullMask, L != 0u);
            const uint32_t nlit = mb ? (uint32_t)__ffs(mb) - 1u : min(32u, seglen - pos);
            if (lane < nlit) { const uint32_t v = win[off + j]; tok[t + lane] = (uint16_t)v; atomicAdd(&s_hist[v], 1u); }
            t += nlit; pos += nlit;
            if (mb) {
                const uint32_t ml = __shfl_sync(kFullMask, L, nlit), md = __shfl_sync(kFullMask, D, nlit);
                if (lane == 0) {
                    tok[t] = (uint16_t)(256u + ml); tok[t + 1] = (uint16_t)(0x8000u | (md - 1u));
                    uint32_t sym, xb, xv;
                    deflate_len_code(ml, sym, xb, xv); atomicAdd(&s_hist[sym], 1u);
                    deflate_dist_code(md, sym, xb, xv); atomicAdd(&s_dhist[sym], 1u);
                }
                t += 2; pos += ml;
            }
        }
        if (lane == 0) p.seg_units[blockIdx.x] = t;
    }
    __syncthreads();
    for (uint32_t i = tid; i < 288; i += blockDim.x) if (s_hist[i]) atomicAdd(&p.hist[(size_t)img * 288 + i], s_hist[i]);
    for (uint32_t i = tid; i < 30; i += blockDim.x) if (s_dhist[i]) atomicAdd(&p.dhist[(size_t)img * 32 + i], s_dhist[i]);
}

// code (LSB-first) and bit count of one token unit under the image's book
__device__ __forceinline__ uint32_t lz_unit_code(uint32_t u, const uint32_t* s_lit, const uint32_t* s_len, const uint32_t* s_dist,
                                                 uint32_t& nbits)
{
    uint32_t e, sym, xb = 0, xv = 0;
    if (u < 256u) e = s_lit[u];
    else if (u < 0x8000u) { deflate_len_code(u - 256u, sym, xb, xv); e = s_len[sym - 257u]; }
    else { deflate_dist_code((u & 0x7FFFu) + 1u, sym, xb, xv); e = s_dist[sym]; }
    const uint32_t sz = e >> 16;
    nbits = sz + xb;
    return (e & 0xFFFFu) | (xv << sz);
}

template <bool PACK>
__global__ void __launch_bounds__(kLzSegThreads) lz_segment_kernel(PngLzParams p)
{
    __shared__ uint32_t s_lit[256], s_len[29], s_dist[30];
    __shared__ unsigned long long s_warp[kLzSegThreads / 32];
    __shared__ uint32_t s_stage[PACK ? kLzStageWords : 1];

    uint32_t seg;
    const uint32_t img = ragged_locate(p.ragged, blockIdx.x, seg);
    if (PACK && p.st[img].stored) return;
    const ImageDesc& d = p.ragged.desc[img];
    const CodeBook* book = d.book;
    const uint32_t tid = threadIdx.x;
    for (uint32_t i = tid; i < 256; i += blockDim.x) s_lit[i] = book->lit[i];
    if (tid < 29) s_len[tid] = book->match[tid];
    if (tid < 30) s_dist[tid] = book->match[32 + tid];
    if (PACK) for (uint32_t i = tid; i < kLzStageWords; i += blockDim.x) s_stage[i] = 0u;
    __syncthreads();

    const uint16_t* tok = p.lz_tok + d.lz_ofs + (unsigned long long)seg * kLzSegment;
    const uint32_t n = p.seg_units[blockIdx.x];
    if (!PACK) {
        unsigned long long bits = 0;
        for (uint32_t i = tid; i < n; i += blockDim.x) { uint32_t nb; lz_unit_code(tok[i], s_lit, s_len, s_dist, nb); bits += nb; }
        unsigned long long tot;
        block_excl_scan_u64(bits, s_warp, tot);
        if (tid == 0) p.seg_bits[blockIdx.x] = (uint32_t)tot;
        return;
    }

    const unsigned long long G = p.seg_ofs[blockIdx.x];
    unsigned long long running = G & 31ull;
    for (uint32_t c = 0; c < n; c += blockDim.x) {
        const uint32_t i = c + tid;
        uint32_t nb = 0, code = 0;
        if (i < n) code = lz_unit_code(tok[i], s_lit, s_len, s_dist, nb);
        unsigned long long tot;
        const unsigned long long at = running + block_excl_scan_u64(nb, s_warp, tot);
        if (nb) {
            const uint32_t w = (uint32_t)(at >> 5), o = (uint32_t)(at & 31ull);
            atomicOr(&s_stage[w], code << o);
            if (o + nb > 32u) atomicOr(&s_stage[w + 1], code >> (32u - o));
        }
        running += tot;
    }
    __syncthreads();
    // whole words out.  A first word that starts mid-word is shared with the previous segment (or the block header), a last word
    // that ends mid-word with the next segment (or the end of block); the offsets kernel zeroed those, so they are OR-ed.  Every
    // other word is this segment's alone and is stored, whatever the output buffer held before.
    uint32_t* file_words = reinterpret_cast<uint32_t*>(p.out + d.out_ofs) + (G >> 5);
    const uint32_t nwords = (uint32_t)((running + 31ull) >> 5);
    for (uint32_t j = tid; j < nwords; j += blockDim.x) {
        const uint32_t v = s_stage[j];
        if ((j == 0 && (G & 31ull)) || (j + 1 == nwords && (running & 31ull))) atomicOr(&file_words[j], v);
        else file_words[j] = v;
    }
}

void launch_lz_match(const PngLzParams& p, uint32_t segs, cudaStream_t s)
{
    FPNGB_SET_SMEM(lz_match_kernel, kLzSmem);
    lz_match_kernel<<<segs, kLzThreads, kLzSmem, s>>>(p);
}

void launch_lz_segments(const PngLzParams& p, uint32_t segs, bool pack, cudaStream_t s)
{
    if (pack) lz_segment_kernel<true><<<segs, kLzSegThreads, 0, s>>>(p);
    else lz_segment_kernel<false><<<segs, kLzSegThreads, 0, s>>>(p);
}

}  // namespace fpngb
