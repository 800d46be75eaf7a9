// fpng_b200/csrc/decode.cuh -- parameter blocks of the decode kernels.
#pragma once
#include "common.cuh"

namespace fpngb {

constexpr int kDecThreads = 256;            // subsequences per CTA in the scan / write kernels
constexpr int kLinkThreads = 1024;          // subsequences linked per step by the per-file chain kernel
constexpr uint32_t kSubBits = 1024;         // bits per subsequence (>> longest token: 12 + 5 + 1 bits)
constexpr uint32_t kPreRoll = 256;          // speculative lead-in before a subsequence (self-synchronisation distance); the
                                            // default of DecodeParams::pre_roll and its maximum (the scan kernel's window lead)

// Per-subsequence record.  After decode_scan_kernel: start/exit/eob_end are absolute aligned-stream bit positions,
// n_out/nlit/lits describe the tokens starting in the subsequence.  decode_link_kernel rewrites it for the write
// kernel: exit := output byte offset, lits := the 4 literals preceding the subsequence, nlit := live flag.
struct SubInfo {
    unsigned long long start, exit, eob_end;
    uint32_t n_out, lits, nlit, pad_;
};

struct FileDesc {                           // filled by the container walk (fpng.cpp:2930-3077), on the host or by container_walk_kernel
    unsigned long long base;                // byte offset of the file from DecodeParams::d_files (a multiple of 4)
    uint32_t file_size, idat_ofs, idat_len;
    uint32_t pre_status;                    // != 0: the file failed before decoding (FPNG_DECODE_* / FPNGB_DECODE_SHAPE_MISMATCH /
                                            // FPNGB_DECODE_OUT_OF_SPACE); no kernel reads its bytes and decode_status_kernel reports this code
    uint32_t w, h, chans;                   // the file's shape: the call's for the uniform calls, the walk's for the ragged call
    uint32_t pitch;                         // bytes per delta row, delta_pitch(w, chans)
    unsigned long long delta_base;          // byte offset of the file's delta rows from DecodeParams::delta (a multiple of 16)
    unsigned long long out_base;            // byte offset of the file's pixel (0, 0, 0) from DecodeParams::d_out
    unsigned long long sub_base;            // index of the file's first record in DecodeParams::subs
};
static_assert(sizeof(FileDesc) == 64, "FileDesc: one 64-byte record per file");

// delta row pitch of a w x chans file, and the number of SubInfo records a file whose IDAT chunk is at most `bytes` long may use
__host__ __device__ __forceinline__ uint32_t delta_pitch(uint32_t w, uint32_t chans) { return (w * chans + 15u) & ~15u; }
__host__ __device__ __forceinline__ uint32_t subs_for(uint32_t bytes) { return (uint32_t)(((uint64_t)bytes * 8 + 32) / kSubBits + 2); }

struct DecodeState {
    uint32_t status;                        // 0 ok, 1 -> FPNG_DECODE_NOT_FPNG; with verification on also the checksum kernels'
                                            // FPNG_DECODE_FAILED_HEADER_CRC32 (4) and FPNGB_DECODE_ADLER_MISMATCH (102)
    uint32_t stored;                        // stored-block file
    unsigned long long token_start;         // bit offset (from the zlib stream start) of the first token
    unsigned long long out_bytes;           // filtered-stream bytes produced
    unsigned long long end_byte;            // bytes consumed up to and including the padded EOB
};

constexpr uint32_t kFastWords = 4096 + 64;   // 4096 fast entries, then the 256 literal code sizes (bytes)

struct DecodeParams {
    const uint8_t* d_files;                 // file f starts at d_files + files[f].base
    const FileDesc* files;                  // [n] device; shape and workspace bases of every file
    DecodeState* state;                     // [n]
    uint32_t* luts;                         // [n][4096]  fused entries, see decode_kernels.cu
    uint32_t* fast;                         // [n][kFastWords]  multi-token entries + literal code sizes of the scan / write loops
    SubInfo* subs;                          // file f: subs + files[f].sub_base, subs_for(idat_len) records at most
    uint8_t* delta;                         // file f: h rows of files[f].pitch bytes at delta + files[f].delta_base (filter byte dropped)
    uint8_t* d_out;                         // pixel (f, y, x, c) at d_out + files[f].out_base + y*row + x*OutStrides::pixel + c*OutStrides::chan
    uint32_t* d_status;                     // [n] FPNG_DECODE_* codes
    uint32_t max_w, max_h, max_subs;        // launch grids: bounds of every file's w, h and subs_for(idat_len)
    uint32_t chans;                         // channels of every file (3 or 4), or 0 when the call mixes both
    uint32_t pre_roll;                      // speculative lead-in bits of decode_scan_kernel, 0..kPreRoll (kPreRoll unless a test sets it)
};

// the rest of the output layout of the decode (unfilter_kernel's second argument; kept out of DecodeParams, which every decode kernel takes)
struct OutStrides {
    size_t row, pixel, chan;                // interleaved (pixel = desired, chan = 1) or planar (pixel = 1); row 0: tight rows of each
                                            // file's own width (w * desired, the ragged call)
};
// Typed output of the decode (fpngb_pixel_format, the *_typed calls): unfilter_typed_kernel stores every value v of output
// channel c as T(__fadd_rn(__fmul_rn(float(v), scale[c]), bias[c])), T = float / __half / __nv_bfloat16 (dtype is the
// FPNGB_DTYPE_* value).  A separate kernel argument, as OutStrides is, so that no other kernel's parameter block grows; the
// OutStrides of a typed call are in bytes, with pixel == sizeof(T) for planar output.
struct PixelAffine { float scale[4], bias[4]; };
// A native call (FPNGB_PNG_NATIVE) is a runtime case of the same kernels: dtype may also be 0 (uint8: the value itself) or
// FPNGB_DTYPE_UINT16 (v * 257, or a 16-bit sample as it is), desired 1..4 or 0 (each file's own channels), and scale / bias act on
// the float types only.
struct TypedOut { uint32_t dtype; PixelAffine aff; };
// Opt-in integrity check of every decode call (fpngb_set_decode_verify).  Two kernels read the file and the delta rows again:
//   idat_crc_stream_kernel<false, true> (crc_stream_kernel.cu), after decode_prepare_kernel: the CRC-32 of "IDAT" + idat_len data
//     bytes against the chunk's CRC field; a mismatch sets DecodeState::status to 4 for every file the walk passed, whatever the
//     stream checks found, so the later kernels skip the file;
//   decode_adler_kernel (decode_kernels.cu), after the write and stored kernels: the Adler-32 of the inflated stream against the
//     stream's last four bytes; a mismatch sets status 102 before unfilter_kernel writes any pixel.
// Their per-file accumulators, zeroed by one cudaMemsetAsync in front of the pipeline:
struct VerifyState {
    uint32_t crc_acc, crc_done;             // XOR of the CRC kernel's CTA contributions, CTAs finished
    uint32_t adler_done, pad_;              // CTAs of the Adler kernel finished
    unsigned long long s1, s2;              // sum x_i and sum i * x_i over the delta rows, each CTA's share reduced mod 65521
};
struct VerifyParams {
    const uint8_t* d_files; const FileDesc* files; DecodeState* state; const uint8_t* delta;   // as in DecodeParams
    VerifyState* vs;                        // [n]
};
// verify: the call's [n] accumulators, or nullptr (verification off: the pipeline is exactly the unverified one);
// max_file_bytes: a bound of every file's size (the CRC kernel's grid); typed: nullptr for uint8 pixels (unfilter_kernel), else the
// output type and affine map of unfilter_typed_kernel, which takes the same launch slot
void launch_decode(const DecodeParams& p, const OutStrides& out, uint32_t n, uint32_t desired, cudaStream_t s,
                   VerifyState* verify = nullptr, size_t max_file_bytes = 0, const TypedOut* typed = nullptr);
// unfilter_typed_kernel (decode_typed_kernels.cu) in launch_decode's unfilter slot, grid g
void launch_unfilter_typed(const DecodeParams& p, const OutStrides& os, const TypedOut& t, uint32_t desired, dim3 g, cudaStream_t s);
void launch_idat_crc_verify(const VerifyParams& p, uint32_t n, size_t max_file_bytes, cudaStream_t s);
void decode_profile_enable(bool on);
int decode_profile_read(float* ms, int n);
unsigned long long decode_link_repairs(bool reset);
bool decode_set_pre_roll(uint32_t bits);    // DecodeParams::pre_roll of later calls; false (unchanged) above kPreRoll

// container_walk_kernel (container_kernels.cu): one thread per file of a packed buffer (d_base + offsets[i], sizes[i] bytes).
// info != nullptr: the six values of fpngb_get_info_ex per file, {status, w, h, chans, idat_ofs, idat_len}.
// files != nullptr: the FileDesc of the packed decode; pre_status holds the argument checks (size 0, size > max_file_size,
// offset % 4, and for the ragged call offset + size > base_bytes), the walk's code, then the shape check:
//   uniform call (chans != 0): FPNGB_DECODE_SHAPE_MISMATCH when a valid file is not w x h x chans; the workspace bases are
//     i * (h * delta_pitch(w, chans)), i * out_stride and i * subs_for(max_file_size);
//   ragged call (chans == 0): the walk runs only when the argument checks pass; with index != 0 FPNGB_DECODE_NOT_INDEXED for a
//     file that has no single sample an element of index bytes holds (include/fpng_b200.h); FPNGB_DECODE_SHAPE_MISMATCH when the file is
//     wider than w or taller than h, FPNG_DECODE_FAILED_DIMENSIONS_TOO_LARGE when w * h * desired > 0xFFFFFFFF, then, for the
//     resized call (boxes != nullptr), FPNGB_DECODE_BAD_CROP when the file's box is empty or not inside the image; the bases are
//     set by decode_place_kernel.
struct WalkParams {
    const uint8_t* base; const unsigned long long* offsets; const uint32_t* sizes; uint32_t n;
    uint32_t* info;                         // [n][6] or nullptr
    FileDesc* files;                        // [n] or nullptr
    uint32_t max_file_size, w, h, chans;    // checks of the `files` output
    uint32_t desired;                       // ragged call: output channels
    unsigned long long base_bytes;          // ragged call: length of the buffer behind base
    unsigned long long out_stride;          // uniform call: output bytes per file
    const int32_t* boxes;                   // resized call: [n][4] {top, left, height, width}, or nullptr (whole images)
    uint32_t index;                         // index call (FPNGB_PNG_INDEX): bytes per output element, 1 or 2; else 0
};
void launch_container_walk(const WalkParams& p, cudaStream_t s);

// decode_place_kernel (container_kernels.cu), ragged call: one CTA places the files the walk accepted, in index order.  File i
// takes align_up(w*h*px_bytes, 16) output bytes, h * pitch delta bytes and subs_for(file_size) records; out_offsets[i] is the
// running output offset (a rejected file takes nothing), out_offsets[n] the total, with bit 63 set when it exceeds out_cap.
// A file whose output, delta rows or records end past out_cap / delta_cap / sub_cap gets FPNGB_DECODE_OUT_OF_SPACE.
struct PlaceParams {
    FileDesc* files; uint32_t n;
    uint32_t px_bytes;                      // output bytes per pixel: desired * sizeof(T) (desired for uint8 pixels); 0 in a native
                                            // call with desired 0: file i's chans * elem
    uint32_t elem;                          // native calls: bytes per element
    unsigned long long out_cap, delta_cap, sub_cap;
    unsigned long long* out_offsets;        // [n + 1]
};
void launch_decode_place(const PlaceParams& p, cudaStream_t s);

// ---- general PNG files (fpngb_decode_packed_png_device, FPNGB_RESIZE_ANY_PNG; png_walk.cuh) ----
// The any-PNG walk gives a general file that passes every check the internal pre_status kPngPending: no fpng kernel touches it and
// decode_status_kernel writes that marker to d_status, which png_unfilter_kernel, launched behind it, overwrites with the file's
// final status.  decode_place_kernel<true> places general files like any file (align_up(w*h*px_bytes, 16) output bytes), takes
// align_up(h * (1 + w*chans), 16) delta bytes for the inflated rows (FileDesc::delta_base) and no records, and allots the gathered
// IDAT bytes (PngDesc::zofs) from a fourth scan bounded by z_cap.
// With FPNGB_PNG_ALL_FORMATS the files png_unfilter_kernel does not read (palette, depth != 8, a color key, Adam7: the "ext" files)
// get kPngPendingExt instead: gather, inflate and place take both markers, png_unfilter_kernel skips them, and png_unfilter_ext_kernel
// writes their final status.  An ext file's inflated bytes are PngDesc::raw_len (delta bytes align_up(raw_len, 16)).
constexpr uint32_t kPngPending = 0x7FFFFFF0u;
constexpr uint32_t kPngPendingExt = 0x7FFFFFF1u;
__host__ __device__ __forceinline__ bool png_pending(uint32_t pre) { return pre == kPngPending || pre == kPngPendingExt; }
struct PngDesc {
    unsigned long long zofs;                // byte offset of the file's gathered zlib stream from PngParams::z (a multiple of 16)
    uint32_t zlen;                          // its length: the sum of the IDAT data lengths
    uint32_t status;                        // 0 until the gather (4) or inflate (8, 102) kernels find an error
    // ext files only (png_walk.cuh's PngFormat; 0 for the others)
    unsigned long long raw_len;             // inflated bytes, every Adam7 pass and filter byte included
    uint32_t depth, type, interlace;        // IHDR bit depth, color type, interlace method
    uint32_t plte_ofs, plte_n;              // PLTE data: offset from the file's first byte, entries
    uint32_t trns_ofs, trns_len;            // tRNS data: offset from the file's first byte (0: none), bytes
    uint32_t pad_;
};
static_assert(sizeof(PngDesc) == 56, "PngDesc");
struct PngParams {
    const uint8_t* d_files; const FileDesc* files; PngDesc* png;
    uint8_t* z;                             // gathered zlib streams
    uint8_t* rows;                          // inflated rows: file f at rows + files[f].delta_base (the decode's delta region)
    uint8_t* d_out; uint32_t* d_status;     // pixels as the ragged decode places them (tight HWC rows at d_out + files[f].out_base)
    uint32_t n, desired, verify;            // desired 0 (native calls only): each file's own channels, FileDesc::chans
    uint32_t index;                         // FPNGB_PNG_INDEX: each pixel's raw sample (desired 1, uint8 or uint16 output)
};
// container_walk_kernel<true> (png != nullptr only with files != nullptr; flags: png_walk's) and decode_place_kernel<true>, z_cap
// the gathered bytes.  In a native call (FPNGB_PNG_NATIVE) WalkParams::desired / PlaceParams::px_bytes may be 0: each file's own
// channel count (its info row's chans) then sizes its output and its FPNG_DECODE_FAILED_DIMENSIONS_TOO_LARGE check.
void launch_container_walk_any(const WalkParams& p, PngDesc* png, uint32_t flags, cudaStream_t s);
void launch_decode_place_any(const PlaceParams& p, PngDesc* png, unsigned long long z_cap, cudaStream_t s);
// gather, inflate and unfilter of the general files (three launches, four with FPNGB_PNG_ALL_FORMATS in flags; grids from n alone),
// behind launch_decode
void launch_png_decode(const PngParams& p, const TypedOut* typed, uint32_t flags, cudaStream_t s);

// decode_resize_kernel (decode_resize_kernels.cu), resized call: after the ragged pipeline has decoded every file into tight uint8
// HWC rows (pitch w * desired) at px + px_offsets[f], crops file f to its box and resizes it to out_h x out_w with the bilinear
// rule of fpngb_decode_packed_resized_device, then stores T(r * scale[c] + bias[c]) (float types) or round_u8(r) (dtype 0).
// Files whose d_status is not 0 are skipped.  Output strides in bytes: element (f, y, x, c) at d_out + f*image + y*row + x*pixel
// + c*chan, interleaved (pixel = desired * sizeof(T)) or planar (pixel = sizeof(T)).  A native call (src_dtype FPNGB_DTYPE_UINT16)
// reads uint16 pixels (pitch w * desired * 2) instead, desired 1 .. 4, and stores the rules of decode_resize_kernels.cu.
// Views call (fpngb_decode_packed_views_device, views != nullptr): output image v (at d_out + v*image, out_h x out_w) is view row v
// instead of file v: its file's box resized to its own size, flipped and placed on the canvas, the stored fill elsewhere; the
// kernel writes view_status[v].  boxes is then unused.
struct ResizeParams {
    const uint8_t* px; const unsigned long long* px_offsets;   // the ragged decode's pixels and their placement
    const FileDesc* files; const int32_t* d_status;
    const int32_t* boxes;                   // [n][4] {top, left, height, width}, or nullptr (whole images)
    uint8_t* d_out;
    unsigned long long image, row, pixel, chan;
    uint32_t out_w, out_h, antialias;
    uint32_t nearest;                       // 0 bilinear, 1 FPNGB_RESIZE_NEAREST, 2 FPNGB_RESIZE_NEAREST_EXACT (decode_nearest_kernel)
    const int32_t* views;                   // [m][10] view rows (include/fpng_b200.h), or nullptr
    int32_t* view_status;                   // [m] with views
    uint32_t n;                             // files: a view's file must be below it
    uint32_t fill[4];                       // with views: per channel, the source value stored outside the placed image
};
void launch_decode_resize(const ResizeParams& p, const TypedOut& t, uint32_t src_dtype, uint32_t m, uint32_t desired, bool cubic,
                          cudaStream_t s);
// profiling (fpngb_decode_profile_read): the start (done false) and end (done true) of the resize kernel, reported in slot 8
void decode_profile_mark_resize(cudaStream_t s, bool done);

}  // namespace fpngb
