// fpng_b200/csrc/crc_stream_kernel.cu -- CRC-32 of a byte stream on the device: the IDAT CRC of the encoders (fpng.cpp:1797-1800
// computes fpng_crc32 over "IDAT" + zlib stream with PCLMULQDQ folding, fpng.cpp:255-281; NVIDIA GPUs have no carry-less
// multiply), the decoder's IDAT check and fpngb_crc32 on host buffers of at least 4 KiB (host_api.cu).
//
// idat_crc_stream_kernel never stages the data and has no barrier in its main loop:
//   * a warp owns 8 KiB of the file; its lanes read consecutive 32-bit words straight from global memory (one coalesced
//     128-byte request per step, 8 independent requests in flight) and each lane runs a Horner recurrence whose step advances
//     the CRC register over 128 bytes (four 256-entry slice tables of that advance in shared memory);
//   * chunks are aligned to the END of the message, so a lane's last word always sits 31 - lane words before the end of its
//     chunk and a warp's chunk sits m * 8 KiB before the end of its CTA's 64 KiB: both multipliers are constants (nibble
//     tables); one modular power per CTA positions the CTA's value in the message; XOR into the image's accumulator; the last
//     CTA of an image appends the (at most 3) bytes after the last whole word, applies init/xorout and stores the CRC.
// The message may start at any byte: the first word's bytes in front of it are masked to zero, which a zero-initialised CRC
// register does not see.  The decoder's opt-in integrity check runs the same kernel over the files it reads (VERIFY).
// About 3.3 thread-instructions per byte (4 table look-ups + 8 address instructions + 3 XORs per word): it replaced a kernel
// that staged 32 KiB tiles in shared memory and combined 128-byte chunk CRCs with a multiply tree, at 7.8 per byte.
#include "kernels.cuh"
#include "crc_math.cuh"
#include "decode.cuh"
#include <algorithm>
#include <cstddef>

namespace fpngb {

constexpr uint32_t kCs2WarpWords = 2048;          // 8 KiB per warp
constexpr uint32_t kCs2Warps = 8;                 // 64 KiB per CTA
constexpr uint32_t kCs2CtaWords = kCs2WarpWords * kCs2Warps;

__device__ uint32_t g2_f128b[4][256];             // byte k of (reg ^ word) advanced over 128 bytes
__device__ uint32_t g2_byte[256];                 // plain byte table (tail bytes)
__device__ uint32_t g2_lane_mul[32][8][16];       // multiply by x^(32 * (32 - lane))
__device__ uint32_t g2_warp_mul[kCs2Warps][8][16];   // multiply by x^(32 * kCs2WarpWords * m)
__constant__ uint32_t c2_xpow2[64];               // x^(2^k)
__device__ uint32_t g2_xpow8[4][256];             // x^(8 * d * 256^k): powers of x by byte digits of the byte distance

int crc_stream_tables_init()
{
    static uint32_t f[4][256], lane[32][8][16], wm[kCs2Warps][8][16], xp[64], p8[4][256];
    static constexpr CrcByteTable t = crc_byte_table();
    crc_advance_tables(f, 128);
    for (uint32_t l = 0; l < 32; l++) crc_mul_table(lane[l], xpow(32ull * (32 - l)));
    for (uint32_t m = 0; m < kCs2Warps; m++) crc_mul_table(wm[m], xpow(32ull * kCs2WarpWords * m));
    crc_xpow2_table(xp);
    for (int k = 0; k < 4; k++) for (unsigned long long d = 0; d < 256; d++) p8[k][d] = xpow(8ull * (d << (8 * k)));
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(g2_f128b, f, sizeof f));
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(g2_byte, t.t, sizeof t.t));
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(g2_lane_mul, lane, sizeof lane));
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(g2_warp_mul, wm, sizeof wm));
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(c2_xpow2, xp, sizeof xp));
    FPNGB_CUDA_OK(cudaMemcpyToSymbol(g2_xpow8, p8, sizeof p8));
    return 0;
}

int crc_stream_table_ptrs(const uint32_t** f128b, const uint32_t** lane_mul)
{
    void *a = nullptr, *b = nullptr;
    FPNGB_CUDA_OK(cudaGetSymbolAddress(&a, g2_f128b));
    FPNGB_CUDA_OK(cudaGetSymbolAddress(&b, g2_lane_mul));
    *f128b = (const uint32_t*)a; *lane_mul = (const uint32_t*)b;
    return 0;
}

// grid (max CTAs per image, n images); only images with st.stored == want_stored (or all when want_stored < 0) are processed.
// RAGGED: a 1-D grid over p.ragged, each image with the CTAs of its own max_encoded_size (crc_stream_ctas_for); its slot in p.out
// is ImageDesc::out_ofs.
// VERIFY: the decoder's check of a file it reads (decode.cuh, VerifyState): file blockIdx.y of p.files, whose message is "IDAT" +
// idat_len data bytes from file byte idat_ofs + 4 (any alignment: ancillary chunks may precede IDAT); the last CTA compares the
// CRC with the chunk's big-endian CRC field and sets the file's status to FPNG_DECODE_FAILED_HEADER_CRC32 when they differ.
static_assert(offsetof(ImageState, tiles_done) == offsetof(ImageState, crc_acc) + 4 &&
              offsetof(VerifyState, crc_done) == offsetof(VerifyState, crc_acc) + 4, "the CTA counter follows the CRC accumulator");
template <bool RAGGED = false, bool VERIFY = false>
using CrcStreamParams = std::conditional_t<VERIFY, VerifyParams, std::conditional_t<RAGGED, RaggedParams<CrcParams>, CrcParams>>;

// MSG_AT (RAGGED only): the message starts at byte ImageDesc::hdr_len - 4 of the file (the files of png_encode_kernels.cu, whose
// header is 41 bytes, or more with a label map's PLTE and tRNS) instead of byte 54
template <bool RAGGED = false, bool VERIFY = false, bool MSG_AT = false>
__global__ void __launch_bounds__(32 * kCs2Warps) idat_crc_stream_kernel(CrcStreamParams<RAGGED, VERIFY> p)
{
    // one copy of the four slice tables (4 KiB).  Eight bank-disjoint copies (32 KiB, lanes l / 4 sharing a copy) were measured:
    // C2 0.380 -> 0.372 ms, but small files (one CTA per file) paid the 8x table fill (C2 G0 0.043 -> 0.064 ms): not kept.
    __shared__ uint32_t s_f[4][256];
    __shared__ uint32_t s_part[kCs2Warps];
    uint32_t img = blockIdx.y, bx = blockIdx.x;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // the message is bytes [m0, L) of the 4-byte aligned buffer file_base()
    uint32_t m0 = kPngHeaderSize - 4u, L;                                   // the message starts at byte 54 ("IDAT")
    [[maybe_unused]] ImageState* st = nullptr;
    auto file_base = [&]() -> const uint8_t* {                               // recomputed where needed rather than kept live
        if constexpr (VERIFY) return p.d_files + p.files[img].base;
        else return p.out + (size_t)img * p.out_stride;
    };
    if constexpr (VERIFY) {
        const FileDesc& fd = p.files[img];
        if (fd.pre_status) return;                                           // never read: the walk or the argument checks failed
        m0 = fd.idat_ofs + 4u; L = m0 + 4u + fd.idat_len;
    } else {
        if constexpr (RAGGED) {
            const uint32_t i = ragged_locate(p.ragged, blockIdx.x, bx);
            p.st += i; p.out += p.ragged.desc[i].out_ofs;
            if constexpr (MSG_AT) m0 = p.ragged.desc[i].hdr_len - 4u;
            img = 0;
        }
        st = p.st + img;
        if (p.stored_only && !st->stored) return;
        L = m0 + 4u + st->zsize;                                             // end of the message (file offset)
    }
    const uint32_t w0 = m0 >> 2;                                             // first word; its bytes before m0 are masked off
    const uint32_t head_mask = 0xFFFFFFFFu << (8u * (m0 & 3u));
    const uint32_t wend = L >> 2;                                            // whole words [w0, wend)
    const uint32_t nwords = wend - w0;
    const uint32_t nctas = (nwords + kCs2CtaWords - 1) / kCs2CtaWords;
    if (bx >= nctas) return;
    for (uint32_t i = tid; i < 1024; i += blockDim.x) (&s_f[0][0])[i] = (&g2_f128b[0][0])[i];
    __syncthreads();

    const uint32_t* fw = reinterpret_cast<const uint32_t*>(file_base());
    // CTA b (counted from the END) covers words [wend - (b+1) * kCs2CtaWords, wend - b * kCs2CtaWords); warp m of it (from the end) 8 KiB
    const long long cta_end = (long long)wend - (long long)bx * kCs2CtaWords;
    const uint32_t m = kCs2Warps - 1u - warp;                                // warps in file order: warp 7 is the last chunk (m = 0)
    const long long chunk_end = cta_end - (long long)m * kCs2WarpWords, chunk_begin = chunk_end - kCs2WarpWords;
    uint32_t c = 0;
    if (chunk_end > (long long)w0) {
        constexpr int kSteps = kCs2WarpWords / 32;                           // 64 lane steps
        constexpr int kBatch = 8;                                            // independent loads in flight per lane
#pragma unroll 1
        for (int k0 = 0; k0 < kSteps; k0 += kBatch) {
            uint32_t w[kBatch];
#pragma unroll
            for (int q = 0; q < kBatch; q++) {
                const long long j = chunk_begin + 32ll * (k0 + q) + lane;
                uint32_t v = 0u;
                if (j >= (long long)w0) {
                    v = __ldg(fw + j);
                    if (j == (long long)w0) v &= head_mask;                 // encoder: bytes 52, 53 are the chunk length field, not part of the message
                }
                w[q] = v;
            }
#pragma unroll
            for (int q = 0; q < kBatch; q++) {
                const uint32_t x = c ^ w[q];
                if (k0 + q + 1 < kSteps) c = s_f[0][x & 0xFFu] ^ s_f[1][(x >> 8) & 0xFFu] ^ s_f[2][(x >> 16) & 0xFFu] ^ s_f[3][x >> 24];
                else c = x;
            }
        }
        c = mul_nibbles(g2_lane_mul[lane], c);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c ^= __shfl_xor_sync(0xFFFFFFFFu, c, o);
    // position the warp's value inside the CTA: m warp chunks follow it (lanes 0..7 look up one nibble each)
    uint32_t part = lane < 8u ? __ldg(&g2_warp_mul[m][lane][(c >> (4u * lane)) & 15u]) : 0u;
    part ^= __shfl_xor_sync(0xFFFFFFFFu, part, 4); part ^= __shfl_xor_sync(0xFFFFFFFFu, part, 2); part ^= __shfl_xor_sync(0xFFFFFFFFu, part, 1);
    if (lane == 0) s_part[warp] = part;
    __syncthreads();
    if (tid == 0) {
        uint32_t acc = 0;
        for (uint32_t u = 0; u < kCs2Warps; u++) acc ^= s_part[u];
        // bx CTAs (64 KiB each) follow this one before the last whole word
        acc = gf2_mulmod(acc, gf2_pow(c2_xpow2, 32ull * kCs2CtaWords * bx));
        // ctr[0]: the message's CRC accumulator, ctr[1]: its CTAs finished
        uint32_t* ctr;
        if constexpr (VERIFY) ctr = &p.vs[img].crc_acc; else ctr = &st->crc_acc;
        atomicXor(ctr, acc);
        __threadfence();
        const uint32_t done = atomicAdd(ctr + 1, 1u);
        if (done == nctas - 1) {
            __threadfence();
            uint32_t reg = atomicXor(ctr, 0u);                               // register after all whole words (zero initial value)
            const uint8_t* fb = file_base();
            for (uint32_t b = wend << 2; b < L; b++) reg = g2_byte[(reg ^ fb[b]) & 0xFFu] ^ (reg >> 8);
            // initial value 0xFFFFFFFF advanced over the whole message (L - m0 bytes), final XOR
            reg ^= gf2_mulmod(0xFFFFFFFFu, gf2_pow(c2_xpow2, 8ull * (L - m0))) ^ 0xFFFFFFFFu;
            if constexpr (VERIFY) {
                const uint8_t* q = fb + L;                                   // the chunk's CRC field
                const uint32_t want = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
                if (reg != want) p.state[img].status = 4u;                   // FPNG_DECODE_FAILED_HEADER_CRC32
            } else {
                uint8_t* q = p.out + (size_t)img * p.out_stride + L;
                q[0] = (uint8_t)(reg >> 24); q[1] = (uint8_t)(reg >> 16); q[2] = (uint8_t)(reg >> 8); q[3] = (uint8_t)reg;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// IDAT CRC from the scanline CRCs of the 16-pixel pack kernel (encode16_kernels.cu): the file is never read back.
//
// The CRC is GF(2)-linear in the message BITS and Deflate packs bits LSB-first, the order the reflected CRC consumes them,
// so the message splits into bit strings whose zero-initialised CRCs are shifted to the end of the message and XOR-ed:
//      "IDAT" + block header | scanline 0 | ... | scanline h-1 | end-of-block code | Adler-32
// A scanline's value R covers its code words at their true word alignment in the file (zero outside its own bits) up to
// word B = ((G + bits) >> 5) + 1: contribution R * x^(E - 32 B), E = end of the message in bits.
// grid (kRowCrcSplit, n): each CTA takes a slice of the image's scanlines; the last CTA of an image adds the fixed parts,
// the initial value and the final XOR (both linear as well) and stores the CRC.
// ------------------------------------------------------------------------------------------------------------------
constexpr uint32_t kRowCrcThreads = 256, kRowCrcSplit = 8;

// x^e from byte-digit tables: x^e = x^(e & 7) * prod_k g2_xpow8[k][digit k of e >> 3]  (e < 2^35: every file this library writes)
__device__ __forceinline__ uint32_t xpow_tab(unsigned long long e)
{
    uint32_t r = kCrcOne >> (uint32_t)(e & 7ull);
    uint32_t d = (uint32_t)(e >> 3);
#pragma unroll 1
    for (int k = 0; d; k++, d >>= 8)
        if (d & 0xFFu) r = gf2_mulmod(r, g2_xpow8[k][d & 0xFFu]);
    return r;
}

// RAGGED: image blockIdx.y of p.desc, with its own CTA count (row_crc_split_for(h)); the grid is sized for the tallest image
template <bool RAGGED = false>
__global__ void __launch_bounds__(kRowCrcThreads) row_crc_combine_kernel(RowCrcParams p)
{
    __shared__ uint32_t s_part[kRowCrcThreads / 32];
    uint32_t img = blockIdx.y, nsplit = gridDim.x;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if constexpr (RAGGED) {
        const ImageDesc& d = p.desc[img];
        p.row_crc += d.row_base; p.row_ofs += d.row_base; p.row_bits += d.row_base; p.books = d.book; p.book_stride = 0;
        p.st += img; p.out += d.out_ofs; p.h = d.h;
        nsplit = min(kRowCrcSplit, (d.h + kRowCrcThreads - 1) / kRowCrcThreads);
        if (blockIdx.x >= nsplit) return;
        img = 0;
    }
    ImageState* st = p.st + img;
    if (st->stored) return;                                                  // stored-block images: idat_crc_stream_kernel reads the file
    const CodeBook* book = p.books + (size_t)img * p.book_stride;
    const unsigned long long E = (unsigned long long)(kPngHeaderSize + st->zsize) * 8ull;
    const size_t r0 = (size_t)img * p.h;
    uint32_t acc = 0;
    for (uint32_t y = blockIdx.x * kRowCrcThreads + tid; y < p.h; y += kRowCrcThreads * nsplit) {
        const unsigned long long B = ((p.row_ofs[r0 + y] + p.row_bits[r0 + y]) >> 5) + 1ull;
        acc ^= gf2_mulmod(p.row_crc[r0 + y], xpow_tab(E - 32ull * B));
    }
    if (blockIdx.x == nsplit - 1) {
        // the fixed parts, one 32-bit piece per thread: block header words, "IDAT", end-of-block code, Adler-32, initial value
        const uint32_t hb = book->hdr_bits, nhw = (hb + 31u) >> 5;
        if (tid < nhw) {
            const uint32_t nb = min(32u, hb - 32u * tid);
            uint32_t v = 0;
            for (uint32_t i = 0; i < (nb + 7u) >> 3; i++) v |= (uint32_t)book->hdr[4u * tid + i] << (8u * i);
            acc ^= gf2_mulmod(crc_bits(0u, v, nb), xpow_tab(E - ((unsigned long long)kZlibBitBase + 32ull * tid + nb)));
        } else if (tid == kRowCrcThreads - 1) {
            acc ^= gf2_mulmod(crc_bits(0u, 0x54414449u, 32), xpow_tab(E - (unsigned long long)kZlibBitBase));   // 'I' 'D' 'A' 'T', first byte in the low bits
        } else if (tid == kRowCrcThreads - 2) {
            const unsigned long long e = p.row_ofs[r0 + p.h - 1] + p.row_bits[r0 + p.h - 1];   // end-of-block code right after the last scanline
            const uint32_t eob_bits = book->eob >> 16;
            acc ^= gf2_mulmod(crc_bits(0u, book->eob & 0xFFFFu, eob_bits), xpow_tab(E - e - eob_bits));
        } else if (tid == kRowCrcThreads - 3) {
            acc ^= crc_bits(0u, __byte_perm(st->adler, 0u, 0x0123), 32);    // Adler-32, big-endian, the last four bytes of the message
        } else if (tid == kRowCrcThreads - 4) {
            acc ^= gf2_mulmod(0xFFFFFFFFu, xpow_tab(E - 8ull * (kPngHeaderSize - 4u))) ^ 0xFFFFFFFFu;   // initial value advanced over the message, final XOR
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc ^= __shfl_xor_sync(0xFFFFFFFFu, acc, o);
    if (lane == 0) s_part[warp] = acc;
    __syncthreads();
    if (tid == 0) {
        acc = 0;
        for (uint32_t u = 0; u < kRowCrcThreads / 32; u++) acc ^= s_part[u];
        atomicXor(&st->crc_acc, acc);
        __threadfence();
        const uint32_t done = atomicAdd(&st->tiles_done, 1u);
        if (done == nsplit - 1) {
            __threadfence();
            const uint32_t crc = atomicXor(&st->crc_acc, 0u);
            uint8_t* q = p.out + (size_t)img * p.out_stride + kPngHeaderSize + st->zsize;
            q[0] = (uint8_t)(crc >> 24); q[1] = (uint8_t)(crc >> 16); q[2] = (uint8_t)(crc >> 8); q[3] = (uint8_t)crc;
        }
    }
}

uint32_t row_crc_split_for(uint32_t h) { return std::min(kRowCrcSplit, (h + kRowCrcThreads - 1) / kRowCrcThreads); }

void launch_row_crc_combine(const RowCrcParams& p, uint32_t n, cudaStream_t s)
{
    const uint32_t split = row_crc_split_for(p.h);
    row_crc_combine_kernel<false><<<dim3(split, n), kRowCrcThreads, 0, s>>>(p);
}

void launch_row_crc_combine_ragged(const RowCrcParams& p, uint32_t n, uint32_t max_split, cudaStream_t s)
{
    row_crc_combine_kernel<true><<<dim3(max_split, n), kRowCrcThreads, 0, s>>>(p);
}

uint32_t crc_stream_ctas_for(size_t max_file_bytes) { return (uint32_t)((max_file_bytes / 4 + kCs2CtaWords - 1) / kCs2CtaWords) + 1u; }

void launch_crc_stream(const CrcParams& p, uint32_t n, size_t max_file_bytes, cudaStream_t s)
{
    dim3 grid(crc_stream_ctas_for(max_file_bytes), n);
    idat_crc_stream_kernel<false><<<grid, 32 * kCs2Warps, 0, s>>>(p);
}

void launch_idat_crc_verify(const VerifyParams& p, uint32_t n, size_t max_file_bytes, cudaStream_t s)
{
    dim3 grid(crc_stream_ctas_for(max_file_bytes), n);
    idat_crc_stream_kernel<false, true><<<grid, 32 * kCs2Warps, 0, s>>>(p);
}

void launch_crc_stream_ragged(const RaggedParams<CrcParams>& p, uint32_t total_ctas, cudaStream_t s)
{
    idat_crc_stream_kernel<true><<<total_ctas, 32 * kCs2Warps, 0, s>>>(p);
}

void launch_crc_stream_png(const RaggedParams<CrcParams>& p, uint32_t total_ctas, cudaStream_t s)
{
    idat_crc_stream_kernel<true, false, true><<<total_ctas, 32 * kCs2Warps, 0, s>>>(p);
}

}  // namespace fpngb
