// fpng_b200/csrc/encode_kernels.cu -- the per-image kernels of the fpng encode pipelines (uniform and ragged; the scan K1 and
// pack K3 kernels are in encode16_kernels.cu):
//
//   K2  row_offsets_kernel  exclusive scan of row bit counts -> row bit offsets; compressed-vs-stored decision
//                           (fpng.cpp:567-588,1705,1728); writes the 58-byte container header, the block header,
//                           EOB, IEND and zeroes the words shared between neighbouring rows
//   K3b adler_finalize_kernel  combines the per-row (S1,S2) partials into the zlib Adler-32 (big-endian)
//
#include "row_walk.cuh"
#include "kernels.cuh"

namespace fpngb {

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
// K3b: Adler-32 combine.  State after row r: a' = a + S1_r, b' = b + n*a + S2_r  (mod 65521), start (1, 0).
// ------------------------------------------------------------------------------------------------
// HDR_LEN (RAGGED only): the zlib stream starts at the image's ImageDesc::hdr_len (the files of png_encode_kernels.cu) instead of
// byte 58
template <bool RAGGED = false, bool HDR_LEN = false>
__global__ void __launch_bounds__(kOffsetsThreads) adler_finalize_kernel(AdlerParams p)
{
    __shared__ unsigned long long s_red[3][kOffsetsThreads / 32];
    uint32_t img = blockIdx.x, zlib_at = kPngHeaderSize;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if constexpr (RAGGED) {                      // image blockIdx.x of p.desc (see row_offsets_kernel)
        const ImageDesc& d = p.desc[img];
        p.row_adler += d.row_base; p.st += img; p.out += d.out_ofs; p.w = d.w; p.h = d.h; p.chans = d.chans;
        if constexpr (HDR_LEN) zlib_at = d.hdr_len;
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
        store_be32(p.out + (size_t)img * p.out_stride + zlib_at + st.zsize - 4u, adler);
        p.st[img].adler = adler;
    }
}

// ------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------
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
    adler_finalize_kernel<true, true><<<n, kOffsetsThreads, 0, s>>>(p);
}

void launch_adler_finalize(const AdlerParams& p, uint32_t n, cudaStream_t s)
{
    adler_finalize_kernel<false><<<n, kOffsetsThreads, 0, s>>>(p);
}

}  // namespace fpngb
