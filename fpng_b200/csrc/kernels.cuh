// fpng_b200/csrc/kernels.cuh -- kernel parameter blocks and launcher prototypes (host_api.cu <-> *_kernels.cu).
#pragma once
#include "common.cuh"
#include <type_traits>

namespace fpngb {

constexpr int kOffsetsThreads = 256;

// One image of a ragged encode call (fpngb_encode_ragged_device): its pixels and shape, where its scanlines sit in the row tables
// and lane records, its code book, its output slot and its container header (the IHDR differs per image).
struct ImageDesc {
    const uint8_t* pixels;
    unsigned long long chan_stride;               // 0: interleaved rows; else planar (see ScanParams)
    unsigned long long row_base;                  // first entry of the image in row_bits / row_adler / row_ofs / row_crc
    unsigned long long lane_base;                 // first lane record (uint2) of the image
    unsigned long long out_ofs;                   // byte offset of the image's slot in the output buffer
    const CodeBook* book;
    uint32_t row_pitch, w, h, chans;
    uint32_t lane_pitch;                          // lane records per scanline: 32 * ceil(w / 512)
    uint32_t index;                               // the image's index in the call (its d_sizes entry)
    uint8_t png_header[kPngHeaderSize];
    uint8_t pad_[2];
    uint32_t hdr_len;                             // PNG call: container header bytes L (41, or 41 + PLTE / tRNS for a label map),
    uint32_t hdr_at;                              // staged at PngEncParams::headers + hdr_at; the zlib stream starts at file byte L
    unsigned long long lz_ofs;                    // LZ77 PNG call: byte offset of the image's filtered stream S in PngEncParams::lz_s
    unsigned long long seg_base;                  // LZ77 PNG call: the image's first segment in the seg_* tables
    uint32_t nseg, pad2_;                         // LZ77 PNG call: segments of S (ceil(N / kLzSegment))
};

// The images one ragged launch covers: CTA b works on image img[j] for the j with cta_start[j] <= b < cta_start[j + 1] (every
// image has at least one CTA), as that image's CTA b - cta_start[j].
struct RaggedWork {
    const ImageDesc* desc;
    const uint32_t* img;                          // [count] indices into desc
    const uint32_t* cta_start;                    // [count] exclusive prefix of the images' CTA counts
    uint32_t count;
};

__device__ __forceinline__ uint32_t ragged_locate(const RaggedWork& rw, uint32_t b, uint32_t& local_cta)
{
    uint32_t lo = 0, hi = rw.count - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (rw.cta_start[mid] <= b) lo = mid; else hi = mid - 1;
    }
    local_cta = b - rw.cta_start[lo];
    return rw.img[lo];
}

struct ScanParams {
    const uint8_t* pixels; size_t image_stride;   // n images
    uint32_t row_pitch;                           // bytes between scanlines
    size_t chan_stride;                           // 0: interleaved pixels; else planar, channel c of pixel x at row + x + c * chan_stride
    uint32_t w, h;
    const CodeBook* books; uint32_t book_stride;  // 0: one shared (1-pass) book, 1: per-image books (2-pass)
    uint32_t* row_bits;                           // [n*h] token bits per row (incl. the filter literal)
    uint2* row_adler;                             // [n*h] (S1, S2) mod 65521 of the filtered row
    ImageState* st;                               // [n]
    uint32_t* hist;                               // [n*288] (histogram mode)
    uint32_t merge_first_unit;                    // RGB 1-pass: filter literal and pixel 0 share a flush unit (fpng.cpp:1187-1203)
    uint2* lane_ofs; uint32_t lane_ofs_pitch;     // [n*h][pitch] per 16-pixel group: .x bit offset inside its row, .y lane_info16()
    uint32_t lit1_rule;                           // 1-pass with an RGBA table under which fpng.cpp:1520-1528 can fire: the launchers
                                                  // take the RGBA kernels' LIT1 instantiations (call-wide: one static RGBA table)
};

struct OffsetsParams {
    const uint32_t* row_bits; unsigned long long* row_ofs;
    const CodeBook* books; uint32_t book_stride;
    ImageState* st;
    uint8_t* out; size_t out_stride; uint32_t* sizes;
    uint32_t w, h, chans, flags;
    uint8_t png_header[kPngHeaderSize];           // IDAT length patched per image on device
    const ImageDesc* desc;                        // ragged kernel: image blockIdx.x's shape, rows, book, slot and header
};

struct PackParams {
    const uint8_t* pixels; size_t image_stride;
    uint32_t row_pitch; size_t chan_stride;       // see ScanParams
    uint32_t w, h;
    const CodeBook* books; uint32_t book_stride;
    const unsigned long long* row_ofs;
    const uint32_t* row_bits;                     // total token bits per row
    const uint2* lane_ofs; uint32_t lane_ofs_pitch;
    uint2* row_adler;                             // rewritten for stored images (raw bytes, filter 0)
    const ImageState* st;
    uint8_t* out; size_t out_stride;
    uint32_t lit1_rule;                           // see ScanParams
    uint32_t stored_only;                         // 16-pixel pack kernel: only write images that fell back to stored blocks (fused encoder ran before)
    // 16-pixel pack kernel: raw CRC-32 of each scanline's code words, computed while they sit in the staging buffer
    // (nullptr = off; the file-reading CRC kernel runs instead).  Tables: crc_stream_kernel.cu.
    uint32_t* row_crc;                            // [n*h]
    const uint32_t* crc_f128b;                    // [4][256] slice tables of the 128-byte advance
    const uint32_t* crc_lane_mul;                 // [32][8][16] nibble tables of x^(32 * (32 - l))
};

// combines the scanline CRCs of the pack kernel into the IDAT CRC (crc_stream_kernel.cu)
struct RowCrcParams {
    const uint32_t* row_crc; const unsigned long long* row_ofs; const uint32_t* row_bits;
    const CodeBook* books; uint32_t book_stride;
    ImageState* st; uint8_t* out; size_t out_stride;
    uint32_t h;
    const ImageDesc* desc;                        // ragged kernel: image blockIdx.y's rows, book, slot and height
};

struct AdlerParams {
    const uint2* row_adler; ImageState* st;
    uint8_t* out; size_t out_stride;
    uint32_t w, h, chans;
    const ImageDesc* desc;                        // ragged kernel: image blockIdx.x's rows, slot and shape
};

struct CrcParams {
    uint8_t* out; size_t out_stride;
    ImageState* st;
    uint32_t stored_only;                         // only images that fell back to stored blocks (the single-pass encoder computed the others' CRC inline)
};

// Parameter block of a ragged scan / hist / pack / stream-CRC launch: the uniform block, whose table pointers are the bases an
// image's row_base / lane_base / index count from, plus the images and CTA map of the launch.  (A separate type, so that the
// uniform kernels' parameter blocks stay as they are.)
template <class P> struct RaggedParams : P { RaggedWork ragged; };

struct HuffParams {
    const uint32_t* hist;                         // [n*288]
    CodeBook* books;                              // [n]
    uint32_t chans;
    uint32_t training;                            // 1: table training (fpng.cpp:909-988): symbol 256 keeps its own count in the scaling
    const ImageDesc* desc;                        // ragged kernel: the channel count of image blockIdx.x
    const uint32_t* dhist;                        // LZ77 PNG books: [n*32] distance-symbol histogram
};

// fpngb_encode_png_ragged_device and fpngb_encode_label_ragged_device (png_encode_kernels.cu): the images are ImageDesc entries
// whose chans is B, the bytes per pixel, whose hdr_len / hdr_at locate the container header in `headers` (signature, IHDR, a label
// map's PLTE and tRNS, the IDAT length and type), and whose chan_stride is the plane stride of a planar image (0: interleaved).
// One block of parameters for every kernel of the pipeline.
struct PngEncParams {
    ImageState* st;                               // [m]
    uint32_t* hist;                               // [m * 288]
    uint8_t* row_filter;                          // [rows] filter type of each scanline
    uint32_t* row_bits;                           // [rows] code bits of each scanline, its filter byte included
    unsigned long long* row_ofs;                  // [rows] file bit offset of each scanline
    uint2* row_adler;                             // [rows] (S1, S2) of the scanline as written
    uint8_t* out; uint32_t* sizes; uint32_t flags;
    const ImageDesc* desc;                        // the images (offsets kernel: image blockIdx.x)
    const uint8_t* headers;                       // the images' container headers (ImageDesc::hdr_at, hdr_len)
    const uint32_t* bad;                          // [call images] nonzero: a label map with an out-of-range id, size 0 (nullptr: none)
    RaggedWork ragged;                            // the images and CTA map of a row-kernel launch
};
// LZ77 mode (FPNGB_LZ77_CHAIN): S, its tokens (one 16-bit unit per byte of S at most, at the same index) and per-segment records.
// (A separate type, so that the other PNG kernels' parameter block stays as it is.)
struct PngLzParams : PngEncParams {
    uint8_t* lz_s;                                // the images' filtered streams (ImageDesc::lz_ofs)
    uint16_t* lz_tok;                             // literal v < 256 | 256 + match length | 0x8000 + distance - 1
    uint32_t* seg_units;                          // [segments] token units of each segment
    uint32_t* seg_bits;                           // [segments] code bits of each segment
    unsigned long long* seg_ofs;                  // [segments] file bit offset of each segment
    uint32_t* dhist;                              // [m * 32] distance-symbol histogram
    uint32_t chain;                               // K: candidates walked per position
};
constexpr uint32_t kLzSegment = 16384;            // bytes of S parsed independently (include/fpng_b200.h, "LZ77")
constexpr uint32_t kLzWindow = 32768;             // largest match distance
uint32_t png_rows_per_cta();
// mode 0: filter choice + histogram, 1: row bits, 2: pack; one launch over the images of one (bpp, depth) class
void launch_png_rows(const PngEncParams& p, uint32_t ctas, uint32_t bpp, uint32_t depth, int mode, cudaStream_t s);
void launch_png_offsets(const PngEncParams& p, uint32_t n, cudaStream_t s);
void launch_huffman_build_png(const HuffParams& p, uint32_t n, cudaStream_t s);
// LZ77 mode: mode 0 filter choice writing S and the row Adler partials, 1 the raw rows of the images that fell back to stored
// blocks; classes also RGB8 (bpp 3) and RGBA8 (bpp 4, depth 8)
void launch_png_lz_rows(const PngLzParams& p, uint32_t ctas, uint32_t bpp, uint32_t depth, int mode, cudaStream_t s);
void launch_png_lz_offsets(const PngLzParams& p, uint32_t n, cudaStream_t s);
void launch_huffman_build_lz(const HuffParams& p, uint32_t n, cudaStream_t s);
// lz77_kernels.cu: one CTA per segment over p.ragged (cta_start: the images' seg_base); match search and greedy parse, then the
// code bits of each segment, then the pack
void launch_lz_match(const PngLzParams& p, uint32_t segs, cudaStream_t s);
void launch_lz_segments(const PngLzParams& p, uint32_t segs, bool pack, cudaStream_t s);
void launch_adler_finalize_png(const AdlerParams& p, uint32_t n, cudaStream_t s);

// opt in to > 48 KiB of dynamic shared memory (per kernel instantiation, once per process)
#define FPNGB_SET_SMEM(kernel, bytes) do { static bool done_ = false; \
    if (!done_) { cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes)); done_ = true; } } while (0)

// third-generation single-pass encoder (encode_fused.cu)
bool fused_eligible(const void* base, size_t image_stride, uint32_t w, uint32_t h, uint32_t chans, uint32_t n);
size_t fused_desc_bytes(uint32_t n, uint32_t w, uint32_t h);
int launch_encode_fused(const uint8_t* pixels, size_t image_stride, uint32_t n, uint32_t w, uint32_t h, uint32_t chans, uint32_t flags,
                        const CodeBook* books, uint32_t book_stride, uint2* row_adler, ImageState* st, void* desc_mem,
                        uint8_t* out, size_t out_stride, uint32_t* sizes, const uint8_t* png_header, uint32_t merge_first_unit, cudaStream_t s,
                        cudaEvent_t mid_event);
void launch_fused_crc(const void* desc_mem, uint32_t n, uint32_t w, uint32_t h, const CodeBook* books, uint32_t book_stride, const ImageState* st,
                      uint8_t* out, size_t out_stride, cudaStream_t s);
int fused_tables_init();
// second-generation IDAT CRC kernel (crc_stream_kernel.cu)
int crc_stream_tables_init();
void launch_crc_stream(const CrcParams& p, uint32_t n, size_t max_file_bytes, cudaStream_t s);
void launch_row_crc_combine(const RowCrcParams& p, uint32_t n, cudaStream_t s);
int crc_stream_table_ptrs(const uint32_t** f128b, const uint32_t** lane_mul);
uint32_t crc_stream_ctas_for(size_t max_file_bytes);     // CTAs of the stream CRC kernel for a file of at most that many bytes
uint32_t row_crc_split_for(uint32_t h);                   // CTAs of the scanline-CRC combine for an image of h scanlines
void launch_crc_stream_ragged(const RaggedParams<CrcParams>& p, uint32_t total_ctas, cudaStream_t s);
void launch_crc_stream_png(const RaggedParams<CrcParams>& p, uint32_t total_ctas, cudaStream_t s);   // message from ImageDesc::hdr_len - 4
void launch_row_crc_combine_ragged(const RowCrcParams& p, uint32_t n, uint32_t max_split, cudaStream_t s);
void launch_offsets_ragged(const OffsetsParams& p, uint32_t n, cudaStream_t s);
void launch_adler_finalize_ragged(const AdlerParams& p, uint32_t n, cudaStream_t s);
void launch_huffman_build_ragged(const HuffParams& p, uint32_t n, cudaStream_t s);

// ragged 16-pixel kernels (encode16_kernels.cu): one launch per (chans, loader) class over `ctas` CTAs (ScanParams::ragged)
enum { kLoad16Staged = 0, kLoad16Direct = 1, kLoad16Planar = 2 };
uint32_t scan16_rows_per_cta();
uint32_t pack16_rows_per_warp(size_t total_rows);        // the uniform launch's rule for a batch of that many scanlines
uint32_t pack16_rows_per_cta(uint32_t rows_per_warp, uint32_t chans);
void launch_scan16_ragged(const RaggedParams<ScanParams>& p, uint32_t ctas, uint32_t chans, int load, cudaStream_t s);
void launch_hist16_ragged(const RaggedParams<ScanParams>& p, uint32_t ctas, uint32_t chans, int load, cudaStream_t s);
void launch_pack16_ragged(const RaggedParams<PackParams>& p, uint32_t ctas, uint32_t chans, int load, uint32_t rows_per_warp, cudaStream_t s);

// Conversion pre-pass (encode_typed_kernels.cu): strided input of T -> tight HWC rows of integer samples.  One descriptor is an
// image, or with n > 1 a batch of n images of one shape: element (i, y, x, c) at src + i*image + y*row + x*pixel + c*chan bytes,
// where pixel is chans * sizeof(T) (interleaved) or sizeof(T) (planar), goes to sample (((i*h + y)*w + x)*chans + c) of
// sample_bytes bytes from byte dst of ConvertParams::dst.  sample_bytes is 1 (uint8) except in the PNG call (2: uint16).
struct ConvDesc {
    const uint8_t* src;
    unsigned long long image, row, chan;          // byte strides (chan: the plane stride of a planar image)
    unsigned long long dst;                       // byte offset of image 0's tight rows
    unsigned long long cta_start;                 // first CTA of the descriptor in the launch
    uint32_t n, w, h, chans;
    uint32_t ctas_per_image;                      // convert_ctas_per_image(w, h)
    uint32_t planar;
    uint32_t sample_bytes;                        // bytes per output sample: 1, or 2 for 16-bit PNG output (png launches only)
};
struct ConvertParams {
    ConvDesc one;                                 // count == 1: the only descriptor, passed by value
    const ConvDesc* desc;                         // count > 1: device table, ascending cta_start
    uint32_t count;
    unsigned long long total_ctas;
    uint8_t* dst;
    float scale[4], bias[4];                      // per channel (the uint8 copy ignores them)
};
enum { kConvInterleaved = 0, kConvPlanar = 1, kConvAny = 2 };   // kConvAny: per descriptor (ConvDesc::planar)
uint32_t convert_ctas_per_image(uint32_t w, uint32_t h);
// dtype: an FPNGB_DTYPE_* value, or 0 for the uint8 copy (kConvInterleaved or kConvPlanar only).  png: the typed PNG call's
// instantiations (a float dtype; 1 to 4 channels and sample_bytes 1 or 2 per descriptor), else 3 or 4 channels of uint8 output.
void launch_convert_pixels(const ConvertParams& p, uint32_t dtype, int layout, bool png, cudaStream_t s);

// Label-map pre-pass (label_pack_kernels.cu): image i's w x h ids (uint8 or int64, `elem` bytes each) at src + y*row + x*pixel bytes are
// range-checked against limit (2^depth for gray, the palette size K for a palette) and packed into rows of `pitch` bytes (a
// multiple of 4) at dst: depth < 16 MSB-first, ceil(w*depth/8) bytes per row, the unused low bits zero; depth 16 native little-endian
// uint16.  An id out of range sets bad[index].  One launch over every image of the call; descriptors ascend in cta_start.
struct LabelDesc {
    const uint8_t* src;
    unsigned long long row, pixel;                // byte strides of the ids
    unsigned long long dst;                       // byte offset of the packed rows in LabelPackParams::dst
    unsigned long long cta_start;                 // first CTA of the image in the launch
    uint32_t w, h, depth, limit;
    uint32_t words;                               // 32-bit output words per row: ceil(w * depth / 32)
    uint32_t index;                               // the image's index in the call (its bad flag)
    uint32_t elem;                                // bytes per id: 1 (uint8) or 8 (int64)
    uint32_t pad_;
};
struct LabelPackParams {
    const LabelDesc* desc; uint32_t count;
    uint8_t* dst;
    uint32_t* bad;
};
uint32_t label_pack_ctas(uint32_t words, uint32_t h);
void launch_label_pack(const LabelPackParams& p, unsigned long long total_ctas, cudaStream_t s);

// Colour-type reduction (reduce_kernels.cu, FPNGB_ENCODE_REDUCE).  Image i's w x h x chans samples of elem bytes (1: uint8, 2: uint16)
// are at src + y*row + x*pixel + c*chan.  The analysis ORs the negative evidence below into ReduceState::flags and collects the
// image's distinct 8-bit RGBA colours (key R << 24 | G << 16 | B << 8 | A; a gray sample g is (g, g, g), a missing alpha 255) in a
// 512-slot open-addressing set.  Slot value 0 means empty, so the colour 0x00000000 is not stored there but kept as kRedHasZero.
enum : uint32_t {
    kRedNotRep8 = 1u,                             // a 16-bit sample is not a multiple of 257
    kRedNotOpaque = 2u,                           // an alpha below its maximum
    kRedNotGray = 4u,                             // a pixel with R, G, B not all equal
    kRedNotL1 = 8u, kRedNotL2 = 16u, kRedNotL4 = 32u,   // an 8-bit gray value off the 1-, 2-, 4-bit lattice (255, 85, 17)
    kRedOverflow = 64u,                           // at least 257 distinct colours
    kRedHasZero = 128u                            // the colour 0x00000000 occurs
};
constexpr uint32_t kReduceSlots = 512;
struct ReduceState { uint32_t flags, count, zero_index, pad_; };     // count: distinct colours (kRedHasZero's included)
struct ReduceTable { uint32_t key[kReduceSlots]; uint8_t index[kReduceSlots]; };   // palette index of key[s] (finalise)
// the read-back of one image: flags and count of its ReduceState, the palette in order (keys as above), K = count entries
struct ReduceResult { uint32_t flags, count, pad_[2]; uint32_t pal[256]; };
struct ReduceDesc {
    const uint8_t* src;
    unsigned long long row, pixel, chan;          // byte strides
    unsigned long long cta_start;                 // first CTA of the image in the analysis launch
    uint32_t w, h, chans, elem;
};
struct ReduceParams {
    const ReduceDesc* desc; uint32_t count;
    ReduceState* st; ReduceTable* tab; ReduceResult* res;
};
uint32_t reduce_analyze_ctas(uint32_t w, uint32_t h);
// the analysis over every image of the call (total_ctas CTAs), then the palette finalise (one CTA per image): two launches
void launch_reduce_analyze(const ReduceParams& p, unsigned long long total_ctas, cudaStream_t s);

// The conversion pre-pass of the images whose format changed: rows of `words` 32-bit words at dst.  mode 0: palette indices (looked up
// in tab) packed MSB-first at `bits` bits; mode 1: gray levels g / step packed the same way; mode 2: tight samples of `bits` output
// channels (source channel j, or chans - 1 for the alpha of a gray+alpha output) at out_bytes bytes (1: the 8-bit value, 2: the
// native uint16).
struct ReduceConvDesc {
    const uint8_t* src;
    unsigned long long row, pixel, chan;
    unsigned long long dst;                       // byte offset of the rows in ReduceConvParams::dst
    unsigned long long cta_start;
    const ReduceTable* tab; const ReduceState* st;
    uint32_t w, h, chans, elem;
    uint32_t mode, bits, out_bytes, step, words, pad_;
};
struct ReduceConvParams { const ReduceConvDesc* desc; uint32_t count; uint8_t* dst; };
uint32_t reduce_convert_ctas(uint32_t words, uint32_t h);
void launch_reduce_convert(const ReduceConvParams& p, unsigned long long total_ctas, cudaStream_t s);

bool walk16_eligible(const void* base, size_t image_stride, uint32_t row_pitch, uint32_t w, uint32_t chans);
void launch_scan16(const ScanParams& p, uint32_t n, uint32_t chans, cudaStream_t s);
void launch_hist16(const ScanParams& p, uint32_t n, uint32_t chans, cudaStream_t s);
void launch_pack16(const PackParams& p, uint32_t n, uint32_t chans, cudaStream_t s);
void set_rows_per_warp16(uint32_t v);          // 0 = automatic (5 scanlines per warp on large batches, 1 otherwise)
void launch_offsets(const OffsetsParams& p, uint32_t n, cudaStream_t s);
void launch_adler_finalize(const AdlerParams& p, uint32_t n, cudaStream_t s);
void launch_huffman_build(const HuffParams& p, uint32_t n, cudaStream_t s);
uint32_t adler_chunk_bytes();
void launch_adler_buffer(const uint8_t* d_buf, size_t n, uint2* d_partials, cudaStream_t s);
// src_offsets: file f at files + src_offsets[f] (multiples of 16), or nullptr: at files + f * stride
void launch_compact(const uint8_t* files, size_t stride, const uint32_t* sizes, uint32_t n, uint8_t* dst, size_t dst_cap,
                    unsigned long long* offsets, cudaStream_t s, const unsigned long long* src_offsets = nullptr);

// host helpers shared by host_api.cu and the tests
uint32_t host_crc32(const void* data, size_t n, uint32_t prev);

}  // namespace fpngb
