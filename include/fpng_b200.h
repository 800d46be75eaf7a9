/*
 * include/fpng_b200.h -- C ABI of the H100-native (sm_90a) fpng hot path (libfpng_b200.so).
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++ or torch types.  The C++ wrappers in
 * include/fpng.h (namespace fpng, same signatures as the reference's src/fpng.h:13-111) and the Python
 * package fpng_b200 are thin layers over these entry points.  Every function cites the reference interface it
 * replaces.  All functions return 0 (FPNGB_OK) on success unless stated otherwise; nothing throws.
 *
 * Error codes: 1..99 = argument/usage errors below; fpngb_decode_* return the reference's FPNG_DECODE_* values
 * (src/fpng.h:57-77) unchanged; 1000 + cudaError_t for CUDA runtime failures.
 */
#ifndef FPNG_B200_H
#define FPNG_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FPNGB_API __attribute__((visibility("default")))

enum {
    FPNGB_OK = 0,
    FPNGB_ERR_INVALID_ARG = 1,       /* reference: fpng_encode_image_to_memory returns false (src/fpng.cpp:1670-1680) */
    FPNGB_ERR_BUFFER_TOO_SMALL = 2,
    FPNGB_ERR_NOT_INITIALIZED = 3,
    FPNGB_ERR_NO_DEVICE = 4,         /* no CUDA device: there is deliberately NO CPU fallback */
    FPNGB_ERR_ALIGNMENT = 5,
    FPNGB_ERR_INTERNAL = 6
};

/* encode flags, bit-compatible with src/fpng.h:34-42 */
enum { FPNGB_ENCODE_SLOWER = 1, FPNGB_FORCE_UNCOMPRESSED = 2 };

/* decode status, value-compatible with src/fpng.h:57-77 */
enum {
    FPNGB_DECODE_SUCCESS = 0, FPNGB_DECODE_NOT_FPNG, FPNGB_DECODE_INVALID_ARG, FPNGB_DECODE_FAILED_NOT_PNG,
    FPNGB_DECODE_FAILED_HEADER_CRC32, FPNGB_DECODE_FAILED_INVALID_DIMENSIONS,
    FPNGB_DECODE_FAILED_DIMENSIONS_TOO_LARGE, FPNGB_DECODE_FAILED_CHUNK_PARSING, FPNGB_DECODE_FAILED_INVALID_IDAT,
    FPNGB_DECODE_FILE_OPEN_FAILED, FPNGB_DECODE_FILE_TOO_LARGE, FPNGB_DECODE_FILE_READ_FAILED,
    FPNGB_DECODE_FILE_SEEK_FAILED
};

/* Replaces fpng::fpng_init() (src/fpng.h:17, src/fpng.cpp:373-376: CPU feature detection).  Here: selects the CUDA
 * device (-1 = current), creates the stream, uploads the static Huffman code books / checksum tables.  Idempotent,
 * thread-safe.  Fails with FPNGB_ERR_NO_DEVICE when no GPU is present. */
FPNGB_API int fpngb_init(int device);
FPNGB_API int fpngb_is_initialized(void);
FPNGB_API const char* fpngb_version(void);

/* Upper bound of the encoded file size for a w x h x chans image: max of the stored-block layout
 * (src/fpng.cpp:1747) and the compressed-path working buffer (src/fpng.cpp:1705), plus header and trailer. */
FPNGB_API size_t fpngb_max_encoded_size(uint32_t w, uint32_t h, uint32_t chans);

/* Replaces fpng::fpng_encode_image_to_memory (src/fpng.h:48, src/fpng.cpp:1662-1803) for HOST buffers:
 * pixels (tightly packed, pitch w*chans, R first) -> PNG file bytes in out[0..*out_size).  out_cap must be at least
 * fpngb_max_encoded_size().  Copies host->device, runs the CUDA kernels, copies the file back; returns after the
 * result is in host memory.  Output is byte-identical to the reference encoder for the same flags. */
FPNGB_API int fpngb_encode_host(const void* pixels, uint32_t w, uint32_t h, uint32_t chans, uint32_t flags,
                                void* out, size_t out_cap, size_t* out_size);

/* Batch of n equally sized images resident in DEVICE memory -> n PNG files in device memory.
 *   d_pixels + i*image_stride : image i (tightly packed rows)
 *   d_out    + i*out_stride   : file i; out_stride >= fpngb_max_encoded_size(), multiple of 16; d_out 16-byte aligned
 *   d_sizes[i]                : file size in bytes (device memory, n x uint32)
 * All kernels are enqueued on `stream` (a cudaStream_t; NULL = the CUDA default stream); the call does not
 * synchronise.  This is the path bench.py times; it is what one rank runs on its shard of a multi-GPU batch. */
FPNGB_API int fpngb_encode_batch_device(const void* d_pixels, size_t image_stride, uint32_t n,
                                        uint32_t w, uint32_t h, uint32_t chans, uint32_t flags,
                                        void* d_out, size_t out_stride, uint32_t* d_sizes, void* stream);

/* ---- Pixel layouts of the *_strided device calls ------------------------------------------------------------------------
 * A batch is an [n, h, w, chans] array of bytes given by a base pointer and four BYTE strides, as a torch tensor reports them:
 * byte (i, y, x, c) is at base + i*image_stride + y*row_pitch + x*pixel_stride + c*chan_stride.  Two layouts are supported:
 *   interleaved: pixel_stride == chans, chan_stride == 1 (HWC rows at any pitch: crops, tiles, padded rows);
 *   planar:      pixel_stride == 1, chan_stride >= 1 (CHW: chan_stride = h*w, row_pitch = w; HCW fits too).
 * The stride of a dimension of size 1 is ignored (w == 1 is interleaved when chan_stride == 1, planar otherwise).  Anything else,
 * such as an RGB view of RGBA pixels (pixel_stride 4, chans 3), and a layout whose last byte overflows the address space, give
 * FPNGB_ERR_INVALID_ARG.  Strides are unsigned: no negative strides.
 *   Encode inputs are only read, so they may overlap (stride 0 for a broadcast batch, tiles whose rows interleave); the row
 *   pitch must be below 2^32.
 *   Decode outputs must not overlap: with the dimensions of size > 1 ordered by stride, each stride is at least the span of
 *   the dimensions below it plus one (stride_k >= sum_{j<k} stride_j * (size_j - 1) + 1).
 * A rejected call enqueues nothing and writes nothing. */

/* fpngb_encode_batch_device with the input in any layout of "Pixel layouts" above: d_pixels and the four strides describe
 * the [n, h, w, chans] batch; everything else as fpngb_encode_batch_device, with the same output bytes as for a tightly packed
 * copy.  The scan and pack kernels read interleaved rows at any pitch and planar images in place; where the batch would
 * go to the opt-in single-pass encoder, it is first copied into the library's workspace by one extra kernel. */
FPNGB_API int fpngb_encode_batch_device_strided(const void* d_pixels, size_t image_stride, size_t row_pitch, size_t pixel_stride,
                                                size_t chan_stride, uint32_t n, uint32_t w, uint32_t h, uint32_t chans, uint32_t flags,
                                                void* d_out, size_t out_stride, uint32_t* d_sizes, void* stream);

/* fpngb_encode_ragged_device: encodes n device images of ANY shapes, channel counts and layouts in one call (a dataset's crops,
 *   thumbnails, scans and frames, one tensor each), into one output buffer.  The shapes are host arguments:
 *     pixels   HOST array of n device addresses; image i's byte (y, x, c) is at pixels[i] + y*row_pitch + x*pixel_stride + c*chan_stride
 *     dims     HOST array of n x {w, h, chans}
 *     strides  HOST array of n x {row_pitch, pixel_stride, chan_stride}, or NULL for tight HWC rows (w*chans, chans, 1)
 *   Each image is one image of "Pixel layouts" above: interleaved rows at any pitch or planar (CHW / HCW); inputs may overlap and
 *   the same pointer may appear more than once.
 *   Output slots: file i goes to d_out + d_out_offsets[i], where the offsets are the exclusive prefix of
 *   align_up(fpngb_max_encoded_size(w_i, h_i, chans_i), 16) in index order and d_out_offsets[n] (device, n+1 entries) is the
 *   total; d_sizes[i] (device) receives the file size.  This is the packed layout fpngb_get_info_batch_device and
 *   fpngb_decode_packed_ragged_device read (base_bytes = d_out_offsets[n]); fpngb_compact_packed_device packs it to exact size.
 *   No byte of d_out past the total is written.  The files are byte-identical to fpngb_encode_batch_device's for each image.
 *   Call-level checks, before anything is enqueued: FPNGB_ERR_INVALID_ARG for n == 0 or n > 65535, a NULL pointer (pixels[i]
 *   included), an image with invalid dimensions or channels, or an unsupported layout; FPNGB_ERR_BUFFER_TOO_SMALL when out_cap
 *   is below the total; FPNGB_ERR_ALIGNMENT unless d_out % 16 == 0.  A rejected call enqueues nothing and writes nothing.
 *   The call is stream-ordered, with no host synchronisation: the per-image descriptors and d_out_offsets go up by
 *   cudaMemcpyAsync from library-owned pinned staging, a ring of buffers each reused only once its last copy has completed.
 *   Launches: per non-empty (chans, loader) class -- 3 or 4 channels times staged / direct / planar loader -- one scan and one
 *   pack kernel, plus one hist kernel with FPNG_ENCODE_SLOWER; then four per-image kernels (offsets, Adler-32, scanline-CRC
 *   combine, stored-block CRC), plus the Huffman build with FPNG_ENCODE_SLOWER.  fpngb_profile_read reports the call in its
 *   usual slots.  Every image takes this route, also under an installed table whose one-pixel-match rule can fire.  The opt-in
 *   single-pass encoder is not used by this call. */
FPNGB_API int fpngb_encode_ragged_device(uint32_t n, const uint64_t* pixels, const uint32_t* dims, const uint64_t* strides, uint32_t flags,
                                         void* d_out, size_t out_cap, uint64_t* d_out_offsets, uint32_t* d_sizes, void* stream);

/* fpngb_encode_png_ragged_device: encodes n device images of 1 to 4 channels and 8 or 16 bits per sample to PNG, in one call and
 *   into the packed layout of fpngb_encode_ragged_device: segmentation masks and mattes (gray8), gray+alpha, depth maps and
 *   16-bit sensor frames (gray16), and 16-bit gray+alpha, RGB and RGBA.
 *     pixels   HOST array of n device addresses
 *     dims     HOST array of n x {w, h, chans, depth}: chans 1..4, depth 8 (uint8 samples) or 16 (native little-endian uint16)
 *     strides  HOST array of n x {row_pitch, pixel_stride, chan_stride} in bytes, or NULL for tight HWC rows; the layouts of
 *              "Pixel layouts" above with elements of depth / 8 bytes (interleaved rows at any pitch, or planar)
 *   Images with depth 8 and 3 or 4 channels are fpng files, encoded exactly as fpngb_encode_ragged_device encodes them with the
 *   same flags (byte-identical), so one call can save a mixed list.  Every other image is written as a PNG that fpng's reader
 *   does not claim (no fdEC chunk): signature, IHDR (color type 0, 4, 2 or 6, no interlace), one IDAT holding a zlib stream
 *   (header 78 01, one dynamic Huffman block built for the image, Adler-32), IEND.  Each row takes the PNG filter with the
 *   smallest sum of min(b, 256 - b) over its filtered bytes (ties to the lower type); runs of equal filtered pixels become
 *   matches at distance B = chans * depth / 8 bytes; the code is fpng's 2-pass construction.  The file falls back to stored
 *   blocks (filter 0 on every row) when that is shorter, or with FPNGB_FORCE_UNCOMPRESSED.  FPNGB_ENCODE_SLOWER only affects
 *   the fpng files.  The exact rules are in DESIGN.md §4.6.
 *   Output slots: file i goes to d_out + d_out_offsets[i], the exclusive prefix of align_up(fpngb_max_encoded_size(w_i, h_i,
 *   B_i), 16) with B_i the bytes per pixel (chans for the fpng files); d_out_offsets[n] is the total, d_sizes[i] the file size.
 *   The bound holds for these files too: their header is 17 bytes shorter than fpng's.  No byte of d_out past the total is written.
 *   Call-level checks, before anything is enqueued: those of fpngb_encode_ragged_device (FPNGB_ERR_INVALID_ARG,
 *   FPNGB_ERR_BUFFER_TOO_SMALL, FPNGB_ERR_ALIGNMENT; FPNGB_ERR_ALIGNMENT also for a 16-bit image whose address or strides are
 *   odd), and FPNGB_ERR_INVALID_ARG for unknown flag bits, a depth other than 8 or 16, chans outside 1..4, and an image whose
 *   slot bound exceeds 2^31 - 1 bytes.  A rejected call enqueues nothing and writes nothing.
 *   Stream-ordered, no host synchronisation; descriptors go up from the pinned staging ring as in fpngb_encode_ragged_device.
 *   Launches: those of fpngb_encode_ragged_device for the fpng images, plus, when the call has other images, three per
 *   non-empty class (gray8, GA8, gray16, GA16, RGB16, RGBA16: filter choice and histogram, row sizes, pack) and four per-image
 *   kernels (Huffman build, offsets, Adler-32, CRC).  fpngb_profile_read reports them in slots 0 (filter and histogram),
 *   1 (Huffman), 2 (row sizes), 3 (offsets), 6 (pack), 7 (Adler-32) and 8 (CRC). */
FPNGB_API int fpngb_encode_png_ragged_device(uint32_t n, const uint64_t* pixels, const uint32_t* dims, const uint64_t* strides,
                                             uint32_t flags, void* d_out, size_t out_cap, uint64_t* d_out_offsets, uint32_t* d_sizes,
                                             void* stream);

/* fpngb_encode_label_ragged_device: encodes n label maps (segmentation class ids, masks) in device memory to palette or gray PNGs
 *   in one call, into the packed layout of fpngb_encode_ragged_device.  Image i is a w x h map of ids v, one of two kinds:
 *     gray     (color type 0) at depth d in {1, 2, 4, 8, 16}; valid ids are 0 <= v < 2^d;
 *     palette  (color type 3) at depth d in {1, 2, 4, 8} with K entries, 1 <= K <= min(256, 2^d); valid ids are 0 <= v < K.
 *     pixels   HOST array of n device addresses
 *     dims     HOST array of n x {w, h, depth, elem}: elem 1 (uint8 ids, depth <= 8) or 8 (int64 ids, e.g. argmax output)
 *     strides  HOST array of n x {row_pitch, pixel_stride} in bytes, or NULL for tight rows (w * elem, elem): the layouts of
 *              "Pixel layouts" above with one channel (any row pitch, stride-0 rows included; 64-bit addressing)
 *     palettes HOST array of n fpngb_label_palette, or NULL: all gray.  entries = 0 means gray; otherwise colors holds entries x
 *              chans bytes in host memory, chans 3 (RGB) or 4 (RGBA).
 *   The file: signature, IHDR (w, h, d, color type, 0, 0, no interlace); for a palette PLTE (K x RGB), then tRNS holding the
 *   alphas of entries 0 .. t-1, t = 1 + the last entry whose alpha is not 255 (no tRNS for an RGB or fully opaque palette); one
 *   IDAT; IEND.  Row bytes: for d < 16 ceil(w*d/8) bytes per row, ids packed MSB-first, the unused low bits of the last byte zero;
 *   for d = 16 big-endian samples.  These rows are encoded exactly as fpngb_encode_png_ragged_device encodes a gray8 image
 *   ceil(w*d/8) pixels wide (a gray16 image for d = 16): filter choice, matches at distance 1 (2), fpng's 2-pass code, the stored
 *   fallback and FPNGB_FORCE_UNCOMPRESSED.  So gray d = 8 from uint8 ids and gray d = 16 from int64 ids give the files
 *   fpngb_encode_png_ragged_device writes for the same uint8 / uint16 image, byte for byte.  DESIGN.md §4.6 "Label maps".
 *   Range check: an image with an id out of range (a negative int64 included) gets d_sizes[i] = 0; nothing outside its slot is
 *   written and every other image of the call is as without it.  The decoders take a size of 0 as FPNGB_DECODE_INVALID_ARG.
 *   Output slots: the exclusive prefix of align_up(fpngb_max_label_encoded_size(w_i, h_i, d_i, palette_i), 16) in d_out_offsets
 *   (n + 1 entries, the last the total); d_sizes[i] the file size.  No byte of d_out past the total is written.
 *   Call-level checks, before anything is enqueued: FPNGB_ERR_INVALID_ARG for flags other than FPNGB_FORCE_UNCOMPRESSED and
 *   FPNGB_LZ77_CHAIN(k),
 *   n outside 1..65535, a NULL pointer, w or h outside 1..2^24, a bad depth, elem, palette size or chans, a palette at depth 16,
 *   an unsupported layout or a slot bound above 2^31 - 1; FPNGB_ERR_BUFFER_TOO_SMALL when out_cap is below the total;
 *   FPNGB_ERR_ALIGNMENT unless d_out % 16 == 0 and each image's address and strides are multiples of elem.  A rejected call
 *   enqueues nothing and writes nothing.  Stream-ordered, no host synchronisation.
 *   Launches: one pre-pass over every image (label_pack_kernel: reads each id once, checks it and writes the packed rows;
 *   fpngb_profile_read slot 9), then the PNG pipeline of fpngb_encode_png_ragged_device on the packed rows. */
typedef struct { const uint8_t* colors; uint32_t entries; uint32_t chans; } fpngb_label_palette;
/* the slot bound: the bound of the packed rows (fpngb_max_encoded_size(ceil(w*d/8), h, 1), or (w, h, 2) for d = 16) plus the
 * PLTE and tRNS chunk bytes of pal (NULL or entries = 0: gray) */
FPNGB_API size_t fpngb_max_label_encoded_size(uint32_t w, uint32_t h, uint32_t depth, const fpngb_label_palette* pal);
FPNGB_API int fpngb_encode_label_ragged_device(uint32_t n, const uint64_t* pixels, const uint32_t* dims, const uint64_t* strides,
                                               const fpngb_label_palette* palettes, uint32_t flags, void* d_out, size_t out_cap,
                                               uint64_t* d_out_offsets, uint32_t* d_sizes, void* stream);

/* ---- colour-type reduction (opt-in: FPNGB_ENCODE_REDUCE on fpngb_encode_png_ragged_device) ----------------------------------
 * With flags & FPNGB_ENCODE_REDUCE every image is written in the smallest PNG format that holds its pixels exactly ("lossless
 * reductions" in PNG optimisers).  For an image of c channels at depth D (8 or 16), over the whole image:
 *   8-bit representable  D = 8, or every sample is a multiple of 257; the samples are then read as v / 257;
 *   opaque               c is 1 or 3, or every alpha is at its maximum;
 *   gray-valued          c is 1 or 2, or R = G = B at every pixel;
 *   lattice depth d      (gray-valued, opaque, 8-bit representable) the least d in {1, 2, 4, 8} such that every gray value is a
 *                        multiple of 255 / (2^d - 1), the values the sub-byte expansion s * 255 / (2^d - 1) of a decoder produces;
 *   K                    the number of distinct 8-bit (R, G, B, A), gray as (g, g, g), a missing alpha as 255 (needed up to 256).
 * The formats that hold the image: gray at depth d, or gray16 (opaque, gray-valued, not 8-bit representable); palette at PIL's
 * depth p(K) (1 for K <= 2, 2 for K <= 4, 4 for K <= 16, else 8; needs 8-bit representable and K <= 256); gray+alpha at D'
 * (gray-valued); RGB at D' (opaque); RGBA at D', where D' is 8 for an 8-bit representable image and 16 otherwise.  The call
 * writes the one with the fewest bits per pixel (d, p(K), 2D', 3D', 4D'), ties in the order gray, palette, gray+alpha, RGB,
 * RGBA.  No trial compression.  A palette lists first the entries whose alpha is below 255, ascending by their big-endian
 * RGBA value, then the opaque entries ascending by RGB, so that tRNS is as short as it can be.
 * The file of an image is byte for byte the file an existing call writes for the reduced input with the same flags:
 *   palette         fpngb_encode_label_ragged_device(index map, the palette as RGBA, depth p(K));
 *   gray, d < 8     fpngb_encode_label_ragged_device(gray / (255 / (2^d - 1)), gray, depth d);
 *   the others      fpngb_encode_png_ragged_device(reduced image): gray8, GA8, gray16, GA16, RGB16 and RGBA16 PNGs, and fpng
 *                   files for RGB8 and RGBA8.
 * FPNGB_ENCODE_SLOWER and FPNGB_FORCE_UNCOMPRESSED keep their meaning.  The fpngb_*_typed calls reject the flag
 * (FPNGB_ERR_INVALID_ARG).  Slot i is sized by fpngb_max_reduced_encoded_size(w_i, h_i, chans_i, depth_i); an image whose bound
 * exceeds 2^31 - 1 is rejected.  The format written is in the file: fpngb_get_info_batch_device reads it back.
 * One host synchronisation: the container header and the row kernels of an image depend on its pixels, so the call enqueues
 * the analysis, reads back each image's flags and palette (1040 bytes per image) and waits for them, with the library's lock
 * held.  Everything after that is enqueued as without the flag; a call without the flag stays stream-ordered and unchanged.
 * Workspace: 3.6 KiB per image (a 512-slot colour set with palette indices, 16 bytes of state, the 1040-byte result and the
 * descriptor), 230 MiB at 65535 images; the reduced rows of the images whose format changed go to the conversion buffer.
 * Launches: two more than the call on the reduced images -- the analysis (one pass over every image; a CTA stops once nothing
 * it could still read would change the format) and the palette finalise (one CTA per image), both in fpngb_profile_read slot
 * 10 -- plus one conversion pre-pass (slot 9) when any image's format changed. */
enum { FPNGB_ENCODE_REDUCE = 256 };
/* the slot bound of FPNGB_ENCODE_REDUCE: the larger of fpngb_max_encoded_size(w, h, chans * depth / 8) and the label bound at
 * depth 8 with a 256-entry palette and a full tRNS (which dominates for small images); every candidate format fits.  0 for chans
 * outside 1..4 or depth other than 8 and 16. */
FPNGB_API size_t fpngb_max_reduced_encoded_size(uint32_t w, uint32_t h, uint32_t chans, uint32_t depth);

/* ---- LZ77 mode (opt-in: FPNGB_LZ77_CHAIN(k) on fpngb_encode_png_ragged_device, its _typed twin and
 * fpngb_encode_label_ragged_device) ---------------------------------------------------------------------------------------------
 * With a chain depth k in 1..256 in the flags, every image of the call, 8-bit RGB and RGBA included (no fpng file is written), is
 * a PNG whose zlib stream holds LZ77 matches at any distance up to 32768, across rows.  The rule (DESIGN.md §4.6 "LZ77"):
 *   S        the filtered stream: per row the filter byte of the row filter rule above, then the filtered row (a label map's or a
 *            reduced image's packed rows as those paths make them).  N = h * (1 + row bytes).
 *   hash     H(p) = ((S[p] << 16 | S[p+1] << 8 | S[p+2]) * 0x9E3779B1 mod 2^32) >> 17, 15 bits.
 *   segments S is cut into segments of 16384 bytes (the last may be shorter), each parsed on its own: no match ends past its
 *            segment's end; sources may lie anywhere earlier in S.
 *   search   at p with p + 3 <= segment end: the earlier positions q with H(q) = H(p), newest first, at most k of them (hash
 *            collisions count), stopping at the first q with p - q > 32768.  A candidate's length is the number of i <
 *            min(258, segment end - p) with S[q+i] = S[p+i] (sources may overlap p).  The longest wins, ties to the nearest;
 *            the walk stops once a candidate reaches the maximum.
 *   parse    greedy: a best length >= 3 emits the match (L, p - q) and advances by L, else the literal S[p] and 1.
 *   code     one dynamic block, BFINAL set, zlib header 78 01.  Literal/length: the 286-symbol histogram with end-of-block counted
 *            once, fpng's 2-pass construction (16-bit scaling, Moffat-Katajainen, limit 12).  Distance: the 30-symbol histogram by
 *            the same construction; with fewer than two distance symbols used, the used symbol s (0 if none) and s ^ 1 get 1-bit
 *            codes.  HDIST is the last distance symbol of nonzero length + 1.  Code-length code as for the other PNG files.
 *   stored   as without the mode: stored blocks (filter 0) when the compressed stream is longer, or with FPNGB_FORCE_UNCOMPRESSED.
 * Containers, slot bounds and offsets are unchanged (the stored fallback bounds every file; RGB8 and RGBA8 use
 * fpngb_max_encoded_size(w, h, 3 | 4)).  It combines with FPNGB_ENCODE_REDUCE and FPNGB_FORCE_UNCOMPRESSED; FPNGB_ENCODE_SLOWER
 * with a chain depth, and a depth above 256, are FPNGB_ERR_INVALID_ARG, checked before anything is enqueued.
 * These files decode through the any-PNG inflate (one warp per file), not fpng's parallel decoder: a single large file decodes
 * more slowly than an fpng file.
 * Launches: per non-empty class a filter pass writing S and a stored-row pass; the match kernel (one CTA per segment:
 * fpngb_profile_read slot 11), the Huffman build, a segment-bits kernel, the offsets, a segment-pack kernel, Adler-32 and CRC.
 * Workspace: about 3 bytes per byte of S (S, one 16-bit token unit per byte at most) plus 16 bytes per segment; a call whose
 * workspace cannot be allocated fails with the CUDA error code, as other calls do. */
#define FPNGB_LZ77_CHAIN(k) ((uint32_t)(k) << 16)

/* Batch of n equally sized images in HOST memory (ideally pinned: see fpngb_host_alloc) -> n files in host memory,
 * out + i*out_stride, sizes[i].  Internally pipelines H2D copy / kernels / D2H copy over chunks of the batch. */
FPNGB_API int fpngb_encode_batch_host(const void* pixels, size_t image_stride, uint32_t n,
                                      uint32_t w, uint32_t h, uint32_t chans, uint32_t flags,
                                      void* out, size_t out_stride, uint32_t* sizes);

/* Replaces fpng::fpng_get_info (src/fpng.h:92, src/fpng.cpp:2930-3083): container walk on the host. */
FPNGB_API int fpngb_get_info(const void* file, uint32_t size, uint32_t* w, uint32_t* h, uint32_t* chans);

/* Replaces fpng::fpng_decode_memory (src/fpng.h:108, src/fpng.cpp:3085-3139) for HOST buffers.  out_cap must be at
 * least w*h*desired (use fpngb_get_info first).  Returns an FPNGB_DECODE_* code. */
FPNGB_API int fpngb_decode_host(const void* file, uint32_t size, void* out, size_t out_cap,
                                uint32_t* w, uint32_t* h, uint32_t* chans, uint32_t desired_chans);

/* Batch decode of n fpng files of identical dimensions/channels resident in DEVICE memory (the device-side
 * counterpart of fpng_decode_memory; what bench.py's decode leg and one rank of a multi-GPU decode run).
 *   d_files + i*file_stride   : file i (file_stride multiple of 4, >= file size + 16; d_files 4-byte aligned)
 *   file_sizes/idat_ofs/idat_len[i] : HOST arrays from the container walk (fpngb_get_info_ex) -- chunk parsing stays on
 *                               the host exactly where the reference does it (src/fpng.cpp:2930-3077)
 *   d_out + i*out_stride      : w*h*desired_chans pixels of file i
 *   d_status[i]               : FPNGB_DECODE_SUCCESS or FPNGB_DECODE_NOT_FPNG (device memory, n x uint32), or with
 *                               fpngb_set_decode_verify(1) also FPNGB_DECODE_FAILED_HEADER_CRC32 / FPNGB_DECODE_ADLER_MISMATCH
 * Enqueued on `stream` (NULL = the CUDA default stream); does not synchronise. */
FPNGB_API int fpngb_decode_batch_device(const void* d_files, size_t file_stride, const uint32_t* file_sizes,
                                        const uint32_t* idat_ofs, const uint32_t* idat_len, uint32_t n,
                                        uint32_t w, uint32_t h, uint32_t chans_in_file, uint32_t desired_chans,
                                        void* d_out, size_t out_stride, uint32_t* d_status, void* stream);
/* fpngb_decode_batch_device writing the pixels in any non-overlapping layout of "Pixel layouts" above (chans = desired_chans):
 * pixel (i, y, x, c) of file i at d_out + i*out_image_stride + y*out_row_pitch + x*out_pixel_stride + c*out_chan_stride.
 * Failed files leave their pixels untouched, as in fpngb_decode_batch_device. */
FPNGB_API int fpngb_decode_batch_device_strided(const void* d_files, size_t file_stride, const uint32_t* file_sizes,
                                                const uint32_t* idat_ofs, const uint32_t* idat_len, uint32_t n,
                                                uint32_t w, uint32_t h, uint32_t chans_in_file, uint32_t desired_chans,
                                                void* d_out, size_t out_image_stride, size_t out_row_pitch,
                                                size_t out_pixel_stride, size_t out_chan_stride, uint32_t* d_status, void* stream);

/* Batch of n fpng files in HOST memory (files[i], sizes[i]; ideally pinned) -> pixels in host memory at out + i*out_stride.
 * Container walk per file on the host (src/fpng.cpp:2930-3077), then H2D / decode kernels / D2H pipelined over chunks.
 * status[i] receives the FPNGB_DECODE_* code of file i; all decodable files must share width/height/channels
 * (returned in *w, *h, *chans).  Batch form of fpng_decode_memory (src/fpng.h:108). */
FPNGB_API int fpngb_decode_batch_host(const void* const* files, const uint32_t* sizes, uint32_t n, uint32_t desired_chans,
                                      void* out, size_t out_stride, uint32_t* w, uint32_t* h, uint32_t* chans, int* status);

/* fpngb_get_info plus the location of the IDAT chunk (offset of the chunk's length field, and the IDAT length). */
FPNGB_API int fpngb_get_info_ex(const void* file, uint32_t size, uint32_t* w, uint32_t* h, uint32_t* chans,
                                uint32_t* idat_ofs, uint32_t* idat_len);

/* ---- files that are already in DEVICE memory, packed back to back (no reference counterpart) -----------------------------
 * File i is the d_sizes[i] bytes at d_base + d_offsets[i]; d_base, d_offsets (n x uint64) and d_sizes (n x uint32) are all
 * device memory.  This is the layout of fpngb_compact_batch_device (n+1 offsets: the last is ignored) and of the window
 * fpngb_gather_encoded_device returns (pass its window, offsets, all_sizes and nranks*nmax; unused slots have size 0).
 * Both calls are stream-ordered on `stream` (NULL = the CUDA default stream): they do no host synchronisation and no host
 * copy of file bytes, offsets or sizes, so no pinned staging is needed.  The container walk runs on the device
 * (container_walk_kernel: one thread per file) and is the same function as the host walk of fpngb_get_info_ex.
 *
 * fpngb_get_info_batch_device: d_info[i*6 + 0..5] = {status, w, h, chans, idat_ofs, idat_len}, the six values
 *   fpngb_get_info_ex returns for file i; a size of 0 gives FPNGB_DECODE_INVALID_ARG.  Any offset alignment.
 *
 * fpngb_decode_packed_device: decodes every file of shape w x h x chans_in_file into d_out + i*out_stride
 *   (w*h*desired_chans bytes).  d_status[i] is what fpng_decode_memory would return for file i (the walk's code, then
 *   FPNGB_DECODE_NOT_FPNG or FPNGB_DECODE_SUCCESS from the decode kernels), with two additions checked in this order:
 *   FPNGB_DECODE_INVALID_ARG for size 0, size > max_file_size or offset % 4 != 0, then, for a file the walk accepts,
 *   FPNGB_DECODE_SHAPE_MISMATCH when its w/h/chans differ from the call's.  The pixels of a file whose status is not 0 are
 *   not written.  max_file_size bounds every decoded file and sizes the decoder's per-file workspace (it replaces the
 *   host-known maximum IDAT length of fpngb_decode_batch_device); fpngb_max_encoded_size(w, h, chans_in_file) always
 *   suffices for files this library or the reference wrote.
 *   Call-level checks as fpngb_decode_batch_device: n <= 65535, the shape limits, out_stride, d_base % 4 == 0.
 *   Memory read: the decode kernels read whole aligned 32-bit words and clamp every read to the last word of the file, so for
 *   a 4-aligned file they stay inside [offset, offset + align_up(size, 4)); the walk reads bytes inside [offset, offset +
 *   size).  The buffer must therefore be readable up to align_up(offset + size, 16) for every file, which the compact and
 *   gather layouts (16-byte aligned files) provide. */
enum { FPNGB_DECODE_SHAPE_MISMATCH = 100 };   /* per-file status of the packed decode only: a valid file of another w/h/chans */
FPNGB_API int fpngb_get_info_batch_device(const void* d_base, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n,
                                          uint32_t* d_info, void* stream);
FPNGB_API int fpngb_decode_packed_device(const void* d_base, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n,
                                         uint32_t max_file_size, uint32_t w, uint32_t h, uint32_t chans_in_file,
                                         uint32_t desired_chans, void* d_out, size_t out_stride, int32_t* d_status, void* stream);
/* fpngb_decode_packed_device writing the pixels in any non-overlapping layout of "Pixel layouts" above, as
 * fpngb_decode_batch_device_strided. */
FPNGB_API int fpngb_decode_packed_device_strided(const void* d_base, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n,
                                                 uint32_t max_file_size, uint32_t w, uint32_t h, uint32_t chans_in_file,
                                                 uint32_t desired_chans, void* d_out, size_t out_image_stride, size_t out_row_pitch,
                                                 size_t out_pixel_stride, size_t out_chan_stride, int32_t* d_status, void* stream);

/* fpngb_decode_packed_ragged_device: decodes packed files of ANY shapes and either channel count in one call (an image dataset's
 *   mixed sizes), with the pixels placed back to back in d_out.  Input layout as above; base_bytes is the length of the buffer
 *   behind d_base.  Per file, in this order, each step only when the earlier ones passed:
 *     1. FPNGB_DECODE_INVALID_ARG for size 0, size > max_file_size, offset % 4 != 0 or offset + size > base_bytes;
 *     2. the container walk (the six values of fpngb_get_info_batch_device go to d_info[i*6 + 0..5] when d_info is not NULL;
 *        a file that failed step 1 is not walked and gets {FPNGB_DECODE_INVALID_ARG, 0, 0, 0, 0, 0});
 *     3. FPNGB_DECODE_SHAPE_MISMATCH when w > max_w or h > max_h, then FPNGB_DECODE_FAILED_DIMENSIONS_TOO_LARGE when
 *        w*h*desired_chans > 0xFFFFFFFF (fpng.cpp:3103-3105);
 *     4. placement: the files that passed take align_up(w*h*desired_chans, 16) bytes each, in index order from offset 0.
 *        d_out_offsets[i] is the running offset (a file that failed earlier gets it too and takes no bytes); d_out_offsets[n] is
 *        the total, with bit 63 set when it exceeds out_cap (retry with that size).  A placed file whose bytes end past out_cap
 *        gets FPNGB_DECODE_OUT_OF_SPACE and is not decoded; the files that fit are a prefix of the placed ones;
 *     5. decode: tight HWC rows (pitch w*desired_chans) at d_out + d_out_offsets[i]; status 0 or FPNGB_DECODE_NOT_FPNG as in
 *        fpngb_decode_packed_device.
 *   The pixels of a file whose status is not 0 are not written, nor is any byte of d_out outside the decoded files.
 *   Call-level checks: FPNGB_ERR_INVALID_ARG unless n <= 65535, desired_chans is 3 or 4, 1 <= max_w, max_h <= 2^24 and
 *   max_file_size > 0; FPNGB_ERR_ALIGNMENT unless d_base % 4 == 0 and d_out % 16 == 0.  A rejected call enqueues nothing and
 *   writes nothing.  The call is stream-ordered: no host synchronisation, no host copy of file bytes, offsets, sizes or shapes.
 *   The workspace is sized from the arguments alone: records from min(base_bytes, n * max_file_size), delta rows from out_cap and
 *   n * max_h (see DESIGN.md section 3); launch grids from max_file_size, max_h and max_w, so tight bounds save launch overhead.
 *   Files that do not overlap always fit the workspace; overlapping ones may get FPNGB_DECODE_OUT_OF_SPACE.
 *   Memory read: as fpngb_decode_packed_device, and no file is read past base_bytes. */
enum { FPNGB_DECODE_OUT_OF_SPACE = 101 };     /* ragged packed decode only: the file's pixels do not fit in out_cap */
FPNGB_API int fpngb_decode_packed_ragged_device(const void* d_base, size_t base_bytes, const uint64_t* d_offsets, const uint32_t* d_sizes,
                                                uint32_t n, uint32_t max_file_size, uint32_t max_w, uint32_t max_h, uint32_t desired_chans,
                                                void* d_out, size_t out_cap, uint64_t* d_out_offsets /* n+1 */, uint32_t* d_info /* n*6 or NULL */,
                                                int32_t* d_status, void* stream);

/* Replace fpng::fpng_crc32 / fpng::fpng_adler32 (src/fpng.h:26-31).  Host buffers.  Buffers of 4 KiB and more are
 * checksummed by the device kernels.  NOTE (the one host-side arithmetic in this library): shorter buffers, and any
 * call made before fpngb_init(), use the small host CRC/Adler routines the container code needs anyway for the 17-byte
 * IHDR and the chunk walk -- a kernel launch for a few dozen bytes would only add latency.  The reference signatures
 * cannot report errors and 0 is a valid checksum, so a device failure is reported on stderr and 0 is returned; use the
 * _ex forms (0 = OK, otherwise an FPNGB_ERR_* / 1000 + cudaError code) to detect failures programmatically. */
FPNGB_API uint32_t fpngb_crc32(const void* data, size_t size, uint32_t prev_crc32);
FPNGB_API uint32_t fpngb_adler32(const void* data, size_t size, uint32_t adler);
FPNGB_API int fpngb_crc32_ex(const void* data, size_t size, uint32_t prev_crc32, uint32_t* out);
FPNGB_API int fpngb_adler32_ex(const void* data, size_t size, uint32_t adler, uint32_t* out);

/* Packs the n variable-size files of a batch (d_files + i*stride, d_sizes[i]) back to back into d_dst, each file
 * starting 16-byte aligned; d_offsets receives n+1 byte offsets (offsets[n] = total; bit 63 of offsets[n] is set when
 * dst_cap was too small -- files that did not fit are not copied).  New (no reference counterpart):
 * the staging step before the single NCCL gather of a rank's encoded shard (BASELINE.json north_star). */
FPNGB_API int fpngb_compact_batch_device(const void* d_files, size_t stride, const uint32_t* d_sizes, uint32_t n,
                                         void* d_dst, size_t dst_cap, uint64_t* d_offsets, void* stream);
/* fpngb_compact_batch_device for files at arbitrary offsets: file i is the d_sizes[i] bytes at d_base + d_src_offsets[i]
 *   (device, n x uint64, each a multiple of 16 -- e.g. the slots of fpngb_encode_ragged_device).  Destination offsets, alignment
 *   and the bit-63 rule are those of fpngb_compact_batch_device; a file whose source offset is not a multiple of 16 is not
 *   copied either, and sets bit 63.  FPNGB_ERR_INVALID_ARG for n == 0, n > 65535 or a NULL pointer; FPNGB_ERR_ALIGNMENT
 *   unless d_base % 16 == 0 and d_dst % 16 == 0.  Stream-ordered, two launches. */
FPNGB_API int fpngb_compact_packed_device(const void* d_base, const uint64_t* d_src_offsets, const uint32_t* d_sizes, uint32_t n,
                                          void* d_dst, size_t dst_cap, uint64_t* d_offsets, void* stream);

/* ---- multi-GPU (SURVEY.md 8b/8e; no reference counterpart: fpng is single-threaded, single-device) ----------------------
 * One process per GPU.  Images shard across ranks with no collective on the data path; afterwards ONE gather brings the
 * encoded files of every rank to the collecting rank (or to every rank).  The communicator is an NCCL communicator on the
 * device given to fpngb_init(): either created here from a ncclUniqueId the caller distributes out of band
 * (fpngb_comm_unique_id on one rank -> any broadcast -> fpngb_comm_init on every rank; collective), or adopted from the
 * caller (fpngb_comm_adopt(ncclComm_t)).
 * fpngb_gather_setup (collective): allocates a receive window of window_bytes on every rank and maps every peer's window
 *   over NVLink (CUDA IPC); max_files_per_rank bounds n_local of the gathers that follow.
 * fpngb_gather_encoded_device (collective, stream-ordered, NO host synchronisation when the peer windows are mapped):
 *   all-gathers the file sizes, derives the packed layout on the device and has every rank store its files directly into
 *   the receiver's window with 128-bit peer stores; a 4-byte all-reduce is the completion barrier.  dst_rank = -1 delivers
 *   to every rank.  Outputs (device pointers owned by the library, valid until the next setup/destroy, to be consumed on
 *   `stream`): *d_window = packed files of all ranks in rank order, each 16-byte aligned; (*d_offsets)[r*nmax + i] = byte
 *   offset of file i of rank r, (*d_offsets)[nranks*nmax] = total bytes (bit 63 set: window too small, files that did
 *   not fit were not copied); (*d_all_sizes)[r*nmax + i] = file size (0 for unused slots).  Without P2P/IPC the same
 *   call falls back to grouped ncclSend/ncclRecv (one host synchronisation for the byte counts); fpngb_comm_info reports
 *   which path is active. */
#define FPNGB_UNIQUE_ID_BYTES 128
FPNGB_API int fpngb_comm_unique_id(void* id128);
FPNGB_API int fpngb_comm_init(const void* id128, int nranks, int rank);
FPNGB_API int fpngb_comm_adopt(void* nccl_comm);
FPNGB_API int fpngb_comm_destroy(void);
FPNGB_API int fpngb_comm_info(int* nranks, int* rank, int* p2p);
FPNGB_API int fpngb_gather_setup(size_t window_bytes, uint32_t max_files_per_rank);
FPNGB_API int fpngb_gather_encoded_device(const void* d_files, size_t stride, const uint32_t* d_sizes, uint32_t n_local, int dst_rank,
                                          void** d_window, uint64_t** d_offsets, uint32_t** d_all_sizes, void* stream);

/* ---- static-table training (reference: FPNG_TRAIN_HUFFMAN_TABLES, fpng_test -t; src/fpng.h:114-120) ----
 * fpngb_train_accumulate_device: adds each image's 16-bit scaled symbol counts (what the reference accumulates in
 *   g_huff_counts, src/fpng.cpp:751-755) to counts[288] (host); the histogram runs in the 2-pass histogram kernel.
 * fpngb_create_dynamic_block_prefix: same outputs as fpng::create_dynamic_block_prefix (src/fpng.cpp:910-988).
 * fpngb_set_static_table: installs such a prefix as the 1-pass table for `chans` (nbytes = 0 restores the built-in one). */
FPNGB_API int fpngb_train_accumulate_device(const void* d_pixels, size_t image_stride, uint32_t n, uint32_t w, uint32_t h,
                                            uint32_t chans, uint64_t* counts288, void* stream);
FPNGB_API int fpngb_create_dynamic_block_prefix(const uint64_t* counts288, uint32_t chans, uint8_t* prefix, size_t prefix_cap,
                                                size_t* prefix_len, uint64_t* bit_buf, int* bit_buf_size,
                                                uint32_t* codes288, uint8_t* sizes288);
FPNGB_API int fpngb_set_static_table(uint32_t chans, const uint8_t* prefix, size_t nbytes, uint32_t bit_buf, uint32_t bit_buf_size);

/* General-PNG fallback hook (SURVEY.md 8f; the reference documents the pattern in src/fpng.h:79-91: "if FPNG_DECODE_NOT_FPNG is
 * returned, fall back to a general purpose PNG decoder").  When a decoder is registered, the C++ wrappers
 * fpng::fpng_decode_memory / fpng_decode_file (include/fpng.h) call it for files the fpng decoder rejects with
 * FPNG_DECODE_NOT_FPNG and return its pixels with FPNG_DECODE_SUCCESS.  The callback returns 0 on success and hands over a
 * malloc()ed buffer of w*h*desired_chans bytes (freed by the library); the C-ABI decode entry points are unaffected and keep
 * returning FPNGB_DECODE_NOT_FPNG.  Pass NULL to unregister. */
typedef int (*fpngb_fallback_decoder)(const void* file, uint32_t size, uint32_t desired_chans, void* user,
                                      void** pixels, uint32_t* w, uint32_t* h, uint32_t* chans_in_file);
FPNGB_API void fpngb_set_fallback_decoder(fpngb_fallback_decoder fn, void* user);
FPNGB_API fpngb_fallback_decoder fpngb_get_fallback_decoder(void** user);

/* ---- opt-in integrity check of the decode (lodepng and pvpng check both sums by default; the reference skips them) ----------
 * The decoder, like the reference, checks the CRC of IHDR and of every ancillary chunk but not the IDAT chunk's CRC-32, and never
 * computes the zlib Adler-32.  A damaged file can then decode to wrong pixels with status 0 when the fpng stream rules still hold
 * (a changed byte inside a stored block; a changed bit that swaps two literal codes of the same length).
 * fpngb_set_decode_verify(1) turns on both checks, on the GPU, in every decode call: fpngb_decode_host, fpngb_decode_batch_host,
 *   fpngb_decode_batch_device(_strided), fpngb_decode_packed_device(_strided), fpngb_decode_packed_ragged_device, and the C++
 *   fpng::fpng_decode_memory / fpng_decode_file.  fpngb_get_info* are unchanged.  One process-wide switch (fpng_decode_memory has
 *   the reference's signature and cannot take a flag), off at load; it may be set before fpngb_init.  A call reads it once,
 *   under the library's lock, when it enqueues.  Default off keeps statuses and pixels those of the reference.
 * Per file, after every earlier status (argument checks, the walk, FPNGB_DECODE_SHAPE_MISMATCH, DIMENSIONS_TOO_LARGE,
 *   FPNGB_DECODE_OUT_OF_SPACE), in this order:
 *     1. the CRC-32 of "IDAT" + the chunk's data against its CRC field: FPNGB_DECODE_FAILED_HEADER_CRC32 (4), the code the walk
 *        gives every other chunk with a bad CRC.  It wins over the stream checks, so a damaged file never comes back as
 *        FPNGB_DECODE_NOT_FPNG, which sends fpng_decode_memory's callers to their general-PNG fallback;
 *     2. FPNGB_DECODE_NOT_FPNG from the stream, as without the check;
 *     3. the Adler-32 of the inflated stream (filter bytes included) against the stream's last four bytes:
 *        FPNGB_DECODE_ADLER_MISMATCH.
 *   A file with status 4 or 102 gets none of its pixels written; the other files of the call decode as with the switch off.
 *   The C++ wrappers do not call the fallback decoder for these two codes.
 * Cost: two more kernels per call (the stream CRC kernel over every file, a pass over the delta rows before the pixels are
 *   written) and one cudaMemsetAsync of 32 bytes per file; fpngb_launch_count grows by 2 per call (per chunk of
 *   fpngb_decode_batch_host), and fpngb_decode_profile_read reports the two kernels in slots 6 (CRC) and 7 (Adler-32).
 *   Still stream-ordered: no host synchronisation is added.  Returns FPNGB_OK; the getter returns 0 or 1. */
enum { FPNGB_DECODE_ADLER_MISMATCH = 102 };   /* verified decode only: the zlib Adler-32 does not match the inflated stream */
FPNGB_API int fpngb_set_decode_verify(int on);
FPNGB_API int fpngb_get_decode_verify(void);

/* ---- typed decode output: float32 / float16 / bfloat16 pixels with a per-channel scale and bias ------------------------------
 * The *_typed calls decode exactly as their uint8 twins and store, for output channel c (0 .. desired_chans-1, counted after
 * the 3 <-> 4 conversion) and v the uint8 value the twin would write (alpha 255 when a 3-channel file is decoded to 4):
 *     out = T( (float)v * scale[c] + bias[c] )
 *   The multiply and the add are two separately rounded fp32 operations (never contracted to an FMA: what numpy and torch eager
 *   compute for x * s + b); T is float32, float16 or bfloat16, converted with round to nearest even, overflow to +-inf (as
 *   torch's .to()).  The conversion runs in the decoder's last kernel, which holds each final pixel in registers: no extra pass
 *   and no uint8 buffer.  Entries of scale / bias at index >= desired_chans are ignored.
 *   Statuses and their order, the verify mode (a file with status 4 or 102 gets no element written), the rule that a failed file's
 *   output is left untouched, the launch count and stream ordering (no host synchronisation) are the uint8 twin's.
 * Call-level checks, in addition to the twin's (a rejected call enqueues nothing and writes nothing):
 *   FPNGB_ERR_INVALID_ARG for a NULL fmt, a dtype other than the three below (uint8 output is the twin itself), or a scale or
 *   bias entry that is not finite (in use: index < desired_chans).
 * fpngb_decode_batch_device_typed / fpngb_decode_packed_device_typed: the arguments of the *_strided twin plus fmt.  All strides
 *   stay in BYTES: element (i, y, x, c) at d_out + i*out_image_stride + y*out_row_pitch + x*out_pixel_stride + c*out_chan_stride.
 *   d_out and every stride must be a multiple of sizeof(T), else FPNGB_ERR_ALIGNMENT; divided by sizeof(T), the strides must form
 *   a non-overlapping interleaved or planar layout of "Pixel layouts" above (pixel_stride == desired_chans * sizeof(T) or
 *   == sizeof(T)), else FPNGB_ERR_INVALID_ARG.
 * fpngb_decode_packed_ragged_device_typed: the arguments of fpngb_decode_packed_ragged_device plus fmt.  File i takes
 *   align_up(w*h*desired_chans*sizeof(T), 16) bytes; d_out_offsets and out_cap are in bytes.  The w*h*desired_chans > 0xFFFFFFFF
 *   rule (FPNGB_DECODE_FAILED_DIMENSIONS_TOO_LARGE) is unchanged, so one file's typed output may pass 4 GiB. */
enum { FPNGB_DTYPE_FLOAT32 = 1, FPNGB_DTYPE_FLOAT16 = 2, FPNGB_DTYPE_BFLOAT16 = 3 };
typedef struct { uint32_t dtype; float scale[4]; float bias[4]; } fpngb_pixel_format;   /* entries >= desired_chans ignored */
FPNGB_API int fpngb_decode_batch_device_typed(const void* d_files, size_t file_stride, const uint32_t* file_sizes,
                                              const uint32_t* idat_ofs, const uint32_t* idat_len, uint32_t n,
                                              uint32_t w, uint32_t h, uint32_t chans_in_file, uint32_t desired_chans,
                                              void* d_out, size_t out_image_stride, size_t out_row_pitch,
                                              size_t out_pixel_stride, size_t out_chan_stride, const fpngb_pixel_format* fmt,
                                              uint32_t* d_status, void* stream);
FPNGB_API int fpngb_decode_packed_device_typed(const void* d_base, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n,
                                               uint32_t max_file_size, uint32_t w, uint32_t h, uint32_t chans_in_file,
                                               uint32_t desired_chans, void* d_out, size_t out_image_stride, size_t out_row_pitch,
                                               size_t out_pixel_stride, size_t out_chan_stride, const fpngb_pixel_format* fmt,
                                               int32_t* d_status, void* stream);
FPNGB_API int fpngb_decode_packed_ragged_device_typed(const void* d_base, size_t base_bytes, const uint64_t* d_offsets,
                                                      const uint32_t* d_sizes, uint32_t n, uint32_t max_file_size, uint32_t max_w,
                                                      uint32_t max_h, uint32_t desired_chans, void* d_out, size_t out_cap,
                                                      uint64_t* d_out_offsets /* n+1 */, uint32_t* d_info /* n*6 or NULL */,
                                                      const fpngb_pixel_format* fmt, int32_t* d_status, void* stream);

/* ---- resized decode: packed files of any shapes into one fixed-size batch, with a per-file crop box ---------------------------
 * fpngb_decode_packed_resized_device decodes the packed files of fpngb_decode_packed_ragged_device, crops file i to its box
 *   d_boxes[i*4 + 0..3] = {top, left, height, width} (device int32; d_boxes NULL: the whole image), resizes the crop to
 *   out_h x out_w with torch's bilinear rule (F.interpolate(mode="bilinear", align_corners=False, antialias=...)) and stores
 *   the batch [n, out_h, out_w, desired_chans]: element (i, y, x, c) at d_out + i*out_image_stride + y*out_row_pitch +
 *   x*out_pixel_stride + c*out_chan_stride, any non-overlapping interleaved or planar layout of "Pixel layouts" (NCHW included).
 * The resize rule, per axis, for a crop length `in`, an output length `out` and output index i; all fp32, as torch's CUDA kernel
 *   (ATen/native/cuda/UpSample.cuh, upsample_antialias::_compute_weights_span / _compute_weights, bilinear filter):
 *     scale   = (float)in / (float)out
 *     aa      = (flags & FPNGB_RESIZE_ANTIALIAS) && scale >= 1
 *     support = aa ? scale : 1;   invscale = aa ? 1 / scale : 1
 *     center  = scale * (i + 0.5f)
 *     xmin    = max((int)(center - support + 0.5f), 0)          (truncation, as torch)
 *     xsize   = min((int)(center + support + 0.5f), in) - xmin
 *     w_j     = tri((j + xmin - center + 0.5f) * invscale), j < xsize, tri(t) = max(0, 1 - |t|); then w_j /= sum(w) if the sum != 0
 *   With support 1 these are exactly the taps and weights of F.interpolate(mode="bilinear", align_corners=False, antialias=False),
 *   edges included.  The resampled value is r = sum_y wy * sum_x wx * p(top + ymin + y, left + xmin + x, c) in fp32, in any
 *   order, where p is the uint8 value fpngb_decode_packed_ragged_device writes (alpha 255 when a 3-channel file is decoded to 4).
 *   Stored: T(__fadd_rn(__fmul_rn(r, scale[c]), bias[c])) for a float fmt (the rule of the *_typed decodes), or, with fmt NULL,
 *   the uint8 cvt.rni.sat.u8.f32(r) (round half to even, clamp to [0, 255]: the typed encode's quantiser).
 * Input: the arguments, bounds (max_file_size, max_w, max_h) and per-file rules of fpngb_decode_packed_ragged_device, and the
 *   verify switch.  pixel_cap bounds the bytes of decoded uint8 pixels the call holds, the sum of align_up(w*h*desired_chans, 16)
 *   over the files it decodes (the ragged call's out_cap; the library keeps these pixels in its own grow-only workspace).
 * Per-file statuses in d_status, in this order, each only when the earlier ones passed: the ragged call's argument checks; the
 *   walk (d_info as in the ragged call); FPNGB_DECODE_SHAPE_MISMATCH, then FPNGB_DECODE_FAILED_DIMENSIONS_TOO_LARGE;
 *   FPNGB_DECODE_BAD_CROP when height or width < 1, top or left < 0, top + height > h or left + width > w (such a file takes
 *   no space and is not decoded); FPNGB_DECODE_OUT_OF_SPACE for a placed file past pixel_cap (the files that fit are a prefix of
 *   the placed ones); the decode (with verify on: 4, then FPNG_DECODE_NOT_FPNG, then 102).  The output slice of a file whose
 *   status is not 0 is left untouched.
 * Call-level checks (a rejected call enqueues nothing and writes nothing): FPNGB_ERR_INVALID_ARG for n == 0 or n > 65535, a NULL
 *   d_base / d_offsets / d_sizes / d_out / d_status, max_file_size == 0, max_w or max_h outside 1..2^24, out_w or out_h outside
 *   1..2^24, desired_chans other than 3 or 4, unknown flags bits, a bad fmt (as the *_typed calls) or a bad layout;
 *   FPNGB_ERR_ALIGNMENT unless d_base % 4 == 0 and d_out and every stride are multiples of the element size.
 * Stream-ordered, no host synchronisation: the ragged pipeline plus one resize kernel, 12 launches (14 with verify on);
 *   fpngb_decode_profile_read reports the resize kernel in slot 8 (slots 6 and 7 are 0 with verify off). */
enum { FPNGB_RESIZE_ANTIALIAS = 1 };
enum { FPNGB_DECODE_BAD_CROP = 103 };   /* resized decode only: the file's crop box is empty or not inside the image */
FPNGB_API int fpngb_decode_packed_resized_device(const void* d_base, size_t base_bytes, const uint64_t* d_offsets, const uint32_t* d_sizes,
                                                 uint32_t n, uint32_t max_file_size, uint32_t max_w, uint32_t max_h, size_t pixel_cap,
                                                 const int32_t* d_boxes /* n x {top, left, height, width}, device, or NULL = whole image */,
                                                 uint32_t out_w, uint32_t out_h, uint32_t desired_chans, uint32_t flags,
                                                 const fpngb_pixel_format* fmt /* NULL = uint8 */,
                                                 void* d_out, size_t out_image_stride, size_t out_row_pitch, size_t out_pixel_stride,
                                                 size_t out_chan_stride, uint32_t* d_info /* n*6 or NULL */, int32_t* d_status, void* stream);

/* ---- general PNG files (any writer) in the packed ragged and resized decodes ---------------------------------------------------
 * The fpng decode reads only files fpng wrote; every other PNG gets FPNGB_DECODE_NOT_FPNG.  The calls below also decode, on the GPU,
 * the PNGs image datasets hold: 8-bit, non-interlaced gray, gray+alpha, RGB and RGBA, from any zlib stream, any mix of the five row
 * filters.  Files the fpng walk accepts take the fpng kernels unchanged; files it rejects with FPNGB_DECODE_NOT_FPNG go to the
 * general walk (the "general files"):
 *   * signature, IHDR length and CRC, the dimension limits, chunk framing and ancillary-chunk CRCs as the fpng walk;
 *   * IHDR must say bit depth 8, color type 0 / 2 / 4 / 6, compression 0, filter method 0, interlace 0, else
 *     FPNGB_DECODE_UNSUPPORTED_PNG (palette, 16-bit, sub-byte depths, Adam7): route such files to a host decoder, or decode them
 *     on the GPU too with FPNGB_PNG_ALL_FORMATS (below);
 *   * FPNGB_DECODE_UNSUPPORTED_PNG also for a critical chunk other than IHDR / PLTE / IDAT / IEND, a second IHDR, a PLTE in a gray
 *     file and a tRNS chunk in a color type 0 or 2 file (whatever desired_chans is); a PLTE in an RGB / RGBA file and every other
 *     ancillary chunk are ignored;
 *   * the IDAT chunks must be consecutive (FPNGB_DECODE_FAILED_CHUNK_PARSING); zero-length ones are legal; no IDAT or fewer than 2
 *     data bytes in all: FPNGB_DECODE_FAILED_INVALID_IDAT.
 *   Info row of a general file: {0, w, h, chans (1 gray, 2 gray+alpha, 3, 4), offset of the first IDAT chunk, sum of the IDAT data
 *   lengths}.  fpng-written files keep fpngb_get_info_ex's row.
 * Stream of a general file (the IDAT payloads concatenated): the zlib header must have CM 8, CINFO <= 7, a correct FCHECK and no
 *   preset dictionary, the Deflate data must be accepted by zlib's inflate up to the end of its final block, inflate to exactly
 *   h * (1 + w * chans) bytes, and every row's filter byte must be <= 4; anything else gives FPNGB_DECODE_FAILED_INVALID_IDAT.
 *   Bytes after the final block are read only with verify on: then, in this order, a bad CRC on any IDAT chunk gives
 *   FPNGB_DECODE_FAILED_HEADER_CRC32 (before any stream check) and a missing or wrong Adler-32 FPNGB_DECODE_ADLER_MISMATCH.
 * Channels: gray Y -> (Y, Y, Y[, 255]); gray+alpha -> (Y, Y, Y[, A]); RGB -> alpha 255 when desired is 4; RGBA -> alpha dropped
 *   when desired is 3 (PIL's convert("RGB") / convert("RGBA")).  Typed output as for fpng files.
 * A file with an fdEC chunk that the fpng walk accepts but whose stream breaks the fpng rules keeps FPNGB_DECODE_NOT_FPNG.
 *
 * fpngb_decode_packed_png_device: fpngb_decode_packed_ragged_device (fmt NULL) or its _typed twin (fmt not NULL) with general files
 *   decoded too.  Same arguments, placement (a general file takes align_up(w*h*desired_chans*elem, 16) bytes, tight HWC rows),
 *   statuses and workspace rules; the workspace also holds each general file's gathered IDAT bytes (at most base_bytes + 16 n for
 *   files that do not overlap) and its inflated rows (inside the delta-row bound).  Three launches more than the ragged call: 14
 *   (16 with verify on).  Stream-ordered, no host synchronisation.
 * fpngb_decode_packed_resized_device with flags & FPNGB_RESIZE_ANY_PNG: the same for the resized call (15 launches, 17 verified);
 *   the crop boxes are checked against the general files' w and h.
 * fpngb_get_info_batch_device with the general rules: fpngb_get_png_info_batch_device (one launch).
 * fpngb_get_png_info: the same walk on the host (arguments as fpngb_get_info_ex). */
enum { FPNGB_DECODE_UNSUPPORTED_PNG = 104 };  /* any-PNG decode: a well-formed PNG this decoder does not read (palette, 16-bit, ...) */
enum { FPNGB_RESIZE_ANY_PNG = 4 };   /* bit 2: flags 2 stays an unknown bit, rejected as before */
FPNGB_API int fpngb_decode_packed_png_device(const void* d_base, size_t base_bytes, const uint64_t* d_offsets, const uint32_t* d_sizes,
                                             uint32_t n, uint32_t max_file_size, uint32_t max_w, uint32_t max_h, uint32_t desired_chans,
                                             void* d_out, size_t out_cap, uint64_t* d_out_offsets /* n+1 */,
                                             uint32_t* d_info /* n*6 or NULL */, const fpngb_pixel_format* fmt /* NULL = uint8 */,
                                             int32_t* d_status, void* stream);
FPNGB_API int fpngb_get_png_info_batch_device(const void* d_base, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n,
                                              uint32_t* d_info, void* stream);
FPNGB_API int fpngb_get_png_info(const void* file, uint32_t size, uint32_t* w, uint32_t* h, uint32_t* chans, uint32_t* idat_ofs,
                                 uint32_t* idat_len);

/* ---- every PNG format in the any-PNG decodes (opt-in: FPNGB_PNG_ALL_FORMATS, FPNGB_RESIZE_ALL_PNG_FORMATS) -----------------------
 * With the flag the general walk also accepts palette, 1/2/4-bit gray, 16-bit, color-keyed (tRNS) and Adam7-interlaced files, and
 * the decode calls decode them on the GPU.  Without it every call behaves as above, FPNGB_DECODE_UNSUPPORTED_PNG included.
 * Walk rules with the flag (host and device):
 *   * IHDR (color type: bit depths) 0: 1, 2, 4, 8, 16; 2: 8, 16; 3: 1, 2, 4, 8; 4: 8, 16; 6: 8, 16; interlace 0 or 1; compression
 *     and filter method 0.  Any other IHDR: FPNGB_DECODE_UNSUPPORTED_PNG.
 *   * PLTE: color type 3 needs exactly one, before the first IDAT, with a length that is a nonzero multiple of 3 and at most 768;
 *     missing, empty, bad length, a second one or one after IDAT: FPNGB_DECODE_FAILED_CHUNK_PARSING.  In a gray file
 *     FPNGB_DECODE_UNSUPPORTED_PNG, in an RGB / RGBA file ignored, as without the flag.
 *   * tRNS: at most one, before the first IDAT, in color type 3 after PLTE; length 2 (type 0), 6 (type 2), at most the palette's
 *     entry count (type 3); any violation: FPNGB_DECODE_FAILED_CHUNK_PARSING.  Ignored in types 4 and 6, as without the flag.
 *   * Unknown critical chunks and a second IHDR: FPNGB_DECODE_UNSUPPORTED_PNG.  Framing, CRC and IDAT-run rules as above.
 *   * Info row: {0, w, h, chans, idat_ofs, idat_len}, chans: gray 1 (2 with tRNS), gray+alpha 2, RGB 3 (4 with tRNS), RGBA 4,
 *     palette 3 (4 with tRNS).  Files fpng wrote keep fpngb_get_info_ex's row and the fpng kernels.
 *   * Inflated size: h * (1 + ceil(w * bits_per_pixel / 8)) without interlace; with Adam7 the sum of that expression over the 7
 *     passes, skipping passes of width or height 0.  Any other size, or a filter byte above 4 in any row of any pass:
 *     FPNGB_DECODE_FAILED_INVALID_IDAT.  With verify on the order of the checks is unchanged: 4, then 8, then 102.
 * Pixel rules (the uint8 value of each output channel):
 *   * gray below 8 bits: Y = s * 255 / (2^d - 1), i.e. s * 255, * 85 or * 17 for d = 1, 2, 4 (libpng's expand, PIL, stb_image);
 *     the padding bits at the end of a row are ignored;
 *   * 16-bit samples: the high byte, s >> 8 (PIL, stb_image, lodepng, libpng's strip_16);
 *   * palette: index i < entry count gives PLTE[i], a larger index (0, 0, 0) (libpng, lodepng; no error); alpha tRNS[i] when i is
 *     below the tRNS length, else 255;
 *   * color key (tRNS in types 0 and 2): alpha 0 when the raw samples equal the key, else 255; the comparison uses full samples
 *     (16 bits in 16-bit files), so a key with bits above the depth never matches;
 *   * then the channel mapping above to desired_chans 3 / 4, applied to the expanded gray / gray+alpha / RGB / RGBA pixel;
 *   * Adam7: every pass pixel lands at its full-image position.
 * Typed output: T(v * scale[c] + bias[c]) as for 8-bit files, v the uint8 value above, except for a 16-bit sample (color or alpha):
 *   there v = s / 257.0f, rounded to nearest (torch's s.float() / 257), so the 8-bit-calibrated normalize_scale_bias stays valid,
 *   257 * k decodes to exactly k, and round(v * 257) == s in float32 for every s.  A color-key alpha and an added alpha are 0 or
 *   255.
 * The resized call resamples the uint8 values above: a 16-bit file is resized from its high bytes.
 * Kernels: one more launch than the any-PNG call without the flag (a warp-per-file unfilter of these files): 15 for the ragged call
 *   (17 with verify on), 16 for the resized call (18).  8-bit gray / gray+alpha / RGB / RGBA files without tRNS or Adam7 take the
 *   kernels of the call without the flag and decode to the same bytes.
 * fpngb_decode_packed_png_device_ex: fpngb_decode_packed_png_device with flags (0 or FPNGB_PNG_ALL_FORMATS; other bits:
 *   FPNGB_ERR_INVALID_ARG).  fpngb_decode_packed_png_device is this call with flags 0.
 * fpngb_decode_packed_resized_device: FPNGB_RESIZE_ALL_PNG_FORMATS is valid only together with FPNGB_RESIZE_ANY_PNG (alone:
 *   FPNGB_ERR_INVALID_ARG).  Bit value 2 stays unknown.
 * fpngb_get_png_info_batch_device_ex / fpngb_get_png_info_ex: the device and host walks with flags (unknown bits: the device call
 *   returns FPNGB_ERR_INVALID_ARG, the host walk FPNGB_DECODE_INVALID_ARG, as for its other argument errors).  Without the _ex
 *   they run with flags 0. */
enum { FPNGB_PNG_ALL_FORMATS = 1 };
enum { FPNGB_RESIZE_ALL_PNG_FORMATS = 8 };

/* ---- native output in the any-PNG ragged decode (opt-in: FPNGB_PNG_NATIVE) -----------------------------------------------------
 * With flags & FPNGB_PNG_NATIVE, fpngb_decode_packed_png_device_ex decodes each file at its own channel count and bit depth:
 * desired_chans may be 0 (each file's own channels), 1, 2, 3 or 4, and fmt may also be FPNGB_DTYPE_UINT16.  Bit values 2 and
 * 0x100 stay unknown; fpngb_get_png_info_*_ex keep rejecting FPNGB_PNG_NATIVE (the walk does not depend on it).
 * Sample domain: files of depth <= 8 work in 8-bit values v (palette entries, sub-byte gray after the scaling above, tRNS alpha);
 *   16-bit files in their 16-bit samples s.  Alpha the file lacks is the domain maximum; a color key gives 0 or the maximum.
 * Storing: uint8 (fmt NULL) stores v, or s >> 8; float stores T(x * scale[c] + bias[c]) with x = v or s / 257 (the rules above);
 *   uint16 (FPNGB_DTYPE_UINT16; scale and bias ignored, as uint8 takes none) stores v * 257, or s.
 * Channels: desired 3 / 4 map as above.  desired 1 / 2: gray -> Y; gray+alpha -> Y or (Y, A); RGB, RGBA and palette -> L or (L, A)
 *   with L = (19595 R + 38470 G + 7471 B + 0x8000) >> 16 in the file's domain (8-bit values for depth <= 8 and palette entries,
 *   16-bit samples for 16-bit files; 32 bits hold it either way).  For 8-bit files this is Pillow's convert("L") / ("LA").
 *   fpng files follow the 8-bit RGB / RGBA rule.  desired 0: file i gets c_i = column 3 of its info row (fpng files 3 or 4).
 * Placement: file i takes align_up(w*h*c_i*elem, 16) bytes, elem 1, 2 or 4; the w*h*desired > 0xFFFFFFFF rule
 *   (FPNG_DECODE_FAILED_DIMENSIONS_TOO_LARGE) uses c_i.  Statuses, their order, untouched failed outputs and the workspace rules
 *   are the call's without the flag.
 * Call-level checks (a rejected call enqueues nothing and writes nothing): FPNGB_ERR_INVALID_ARG for desired_chans above 4 or a bad
 *   float fmt; FPNGB_ERR_ALIGNMENT for d_out % 16 as without the flag.  Without FPNGB_PNG_NATIVE every call keeps rejecting dtype
 *   FPNGB_DTYPE_UINT16 (the *_typed calls included) and desired_chans other than 3 and 4.
 * Kernels: the launches of the call without the flag, none added; desired 3 / 4 in uint8 and float give that call's bytes.
 *
 * fpngb_decode_packed_resized_device with flags & FPNGB_RESIZE_NATIVE (valid only together with FPNGB_RESIZE_ANY_PNG; alone:
 *   FPNGB_ERR_INVALID_ARG; bits 2 and 8-alone stay rejected): desired_chans 1 .. 4 (0 is rejected: the batch has one shape), fmt
 *   as above (NULL uint8, FPNGB_DTYPE_UINT16, or a float type).
 *   * The ragged decode behind the resize holds every file as uint16 values of the desired channels, in the 16-bit domain above
 *     (8-bit values v as v * 257); pixel_cap counts the bytes of that intermediate, align_up(w*h*desired_chans*2, 16) per file.
 *   * The resample r runs on those values with the taps and weights above, and stores cvt.rni.sat.u16.f32(r) for uint16,
 *     round_u8(r / 257) for uint8 and T((r / 257) * scale[c] + bias[c]) for a float fmt, every operation separately rounded.
 *   * So a 16-bit file is resized from its full samples.  For an 8-bit file r / 257 may differ from the flag-off r in the last
 *     float bit (the resample runs on 257 times the values), so float output may differ in its last bit from the call without
 *     the flag; uint8 output may differ by one where r sits within that bit of a rounding tie.
 *   * Launches, statuses and stream ordering are the call's without the flag. */
enum { FPNGB_PNG_NATIVE = 4 };
enum { FPNGB_DTYPE_UINT16 = 4 };
enum { FPNGB_RESIZE_NATIVE = 16 };
FPNGB_API int fpngb_decode_packed_png_device_ex(const void* d_base, size_t base_bytes, const uint64_t* d_offsets, const uint32_t* d_sizes,
                                                uint32_t n, uint32_t max_file_size, uint32_t max_w, uint32_t max_h, uint32_t desired_chans,
                                                void* d_out, size_t out_cap, uint64_t* d_out_offsets /* n+1 */,
                                                uint32_t* d_info /* n*6 or NULL */, uint32_t flags,
                                                const fpngb_pixel_format* fmt /* NULL = uint8 */, int32_t* d_status, void* stream);

FPNGB_API int fpngb_get_png_info_batch_device_ex(const void* d_base, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n,
                                                 uint32_t flags, uint32_t* d_info, void* stream);
FPNGB_API int fpngb_get_png_info_ex(const void* file, uint32_t size, uint32_t flags, uint32_t* w, uint32_t* h, uint32_t* chans,
                                    uint32_t* idat_ofs, uint32_t* idat_len);
/* test hook: png_raw_len, the inflated size above, of a w x h file of bits_per_pixel bits (1..64) and interlace method 0 / 1 */
FPNGB_API uint64_t fpngb_debug_png_raw_len(uint32_t w, uint32_t h, uint32_t bits_per_pixel, uint32_t interlace);

/* ---- label maps: raw sample output (opt-in: FPNGB_PNG_INDEX, FPNGB_RESIZE_INDEX) and nearest-neighbour resize ------------------
 * A label map stores class or instance ids, not colours: a palette file's indices (PASCAL VOC, PIL mode "P"), 1-bit masks (PIL
 * mode "1"), 8- or 16-bit gray id maps (Cityscapes *_instanceIds.png).  With flags & FPNGB_PNG_INDEX, fpngb_decode_packed_png_device_ex
 * stores each file's one raw sample per pixel:
 *   * valid only together with FPNGB_PNG_ALL_FORMATS | FPNGB_PNG_NATIVE, desired_chans 1 and fmt NULL (uint8) or
 *     FPNGB_DTYPE_UINT16; anything else (a float fmt included: ids are not scaled) gives FPNGB_ERR_INVALID_ARG.  Bits 2 and 0x100
 *     stay unknown; fpngb_get_png_info_*_ex keep rejecting FPNGB_PNG_INDEX (the walk does not depend on it; info rows unchanged).
 *   * Pixel rule: the sample as stored, with no scaling, no palette lookup and no alpha.  Color type 3: the palette index (an index
 *     at or past the entry count is stored as it is; tRNS ignored).  Color type 0, any depth: the gray sample s (1-bit: 0 / 1,
 *     4-bit: 0..15; a color key ignored).  Adam7 pixels land at their image positions.  For palette files and 8-bit gray this is
 *     np.asarray(PIL.Image.open(f)); for mode "1" that array as uint8; for 2- and 4-bit gray PIL scales the samples, this rule
 *     does not.
 *   * FPNGB_DECODE_NOT_INDEXED (per file) for a file with no single sample the output type holds: fpng files, color types 2, 4
 *     and 6, and a 16-bit gray file decoded to uint8 (it is not truncated).  It comes right after a successful walk, before the
 *     shape, size, crop and space checks; such a file takes no output space, is not decoded, and its output bytes are left
 *     untouched.  Its info row is written as usual.
 *   * Placement: file i takes align_up(w*h*elem, 16) bytes, elem 1 or 2.  Launches: those of the ALL_FORMATS | NATIVE call, none
 *     added (8-bit gray files without tRNS or Adam7 keep the 8-bit unfilter kernel, the others take the ext files' one).
 *
 * fpngb_decode_packed_resized_device with flags & FPNGB_RESIZE_NEAREST or FPNGB_RESIZE_NEAREST_EXACT resizes by nearest neighbour
 * instead of bilinearly: torch's F.interpolate(mode="nearest") / ("nearest-exact"), torchvision's InterpolationMode.NEAREST /
 * NEAREST_EXACT.  Either flag goes with every other flag combination except FPNGB_RESIZE_ANTIALIAS; both together, or either one
 * with FPNGB_RESIZE_ANTIALIAS, give FPNGB_ERR_INVALID_ARG (torch has no antialiased nearest).  Bit 2, and 8 without 4, stay rejected.
 *   * Rule per axis, crop length `in`, output length `out`, output index i, all fp32 and separately rounded (torch's CUDA kernel,
 *     ATen/native/cuda/UpSample.cuh):
 *         scale = (float)in / (float)out
 *         nearest:        src = min((int)floorf((float)i * scale), in - 1)
 *         nearest-exact:  src = min((int)floorf(((float)i + 0.5f) * scale), in - 1)
 *   * Stored value: element (y, x, c) of file i's slice is, bit for bit, what the ragged decode with the same flags, dtype, scale
 *     and bias stores at source pixel (top + src_y, left + src_x).  A native call gathers from the uint16 intermediate u and stores
 *     u >> 8 for uint8, u for uint16 and T(__fdiv_rn(u, 257) * scale[c] + bias[c]) for a float fmt, the native ragged element;
 *     other calls store the uint8 value or its typed conversion.  At identity size nearest is the ragged decode cropped to the
 *     box.  So native uint8 output of a 16-bit file is s >> 8 here, not the bilinear path's round_u8(s / 257).
 *   * FPNGB_RESIZE_INDEX: the FPNGB_PNG_INDEX rule above in the resized call.  It needs FPNGB_RESIZE_ANY_PNG |
 *     FPNGB_RESIZE_ALL_PNG_FORMATS | FPNGB_RESIZE_NATIVE, a nearest flag, desired_chans 1 and fmt NULL or FPNGB_DTYPE_UINT16; anything
 *     else gives FPNGB_ERR_INVALID_ARG (bilinear on ids is refused).  The intermediate has the output's element type, and pixel_cap
 *     counts align_up(w*h*elem, 16) per file.  FPNGB_DECODE_NOT_INDEXED as above; FPNGB_DECODE_BAD_CROP comes after it.
 *   * Launches are those of the call without the flag: decode_nearest_kernel takes decode_resize_kernel's place, and
 *     fpngb_decode_profile_read reports it in slot 8. */
enum { FPNGB_PNG_INDEX = 8 };
enum { FPNGB_DECODE_NOT_INDEXED = 105 };   /* index decode: the file has no single sample the output type holds */
enum { FPNGB_RESIZE_NEAREST = 32, FPNGB_RESIZE_NEAREST_EXACT = 64, FPNGB_RESIZE_INDEX = 128 };

/* ---- views: any number of output images per call, each a crop of a file resized to its own size, flipped and placed ----------
 * fpngb_decode_packed_views_device decodes the packed files as fpngb_decode_packed_resized_device does, then writes m output images
 * ("views") of one canvas size out_h x out_w: element (v, y, x, c) at d_out + v*out_image_stride + y*out_row_pitch +
 * x*out_pixel_stride + c*out_chan_stride, any layout of "Pixel layouts".  A view reads one file; a file may have any number of
 * views, or none.  The view table d_views is a device int32 [m][10], row v = {file, top, left, height, width, resize_h, resize_w,
 * offset_y, offset_x, flags}, flags a combination of FPNGB_VIEW_HFLIP and FPNGB_VIEW_VFLIP.  For view v of file f:
 *   1. R = what fpngb_decode_packed_resized_device stores for file f with box {top, left, height, width}, out_h x out_w :=
 *      resize_h x resize_w, and this call's flags, fmt, interpolation and native / index mode (every rule of that call applies);
 *   2. R' = R with column j taken from resize_w - 1 - j (HFLIP) and row i from resize_h - 1 - i (VFLIP): flips act after the
 *      resize, as an index map, so the taps and weights of each resized value are unchanged;
 *   3. out[v, y, x, c] = R'[y - offset_y, x - offset_x, c] where that position lies inside R', else the fill: fill[c] taken as a
 *      source value of the call and stored as the call stores one (uint8: as it is; float: T(fill * scale + bias); native: a
 *      16-bit domain value under the native store rules of the interpolation; index: the raw sample, e.g. 255 for "ignore").
 *   The result is bit-identical to the resized call at resize_h x resize_w, then the flip, then a paste into a filled canvas: the
 *   accumulation order of each resized value depends neither on the tile nor on the placement.
 * Fill: fill (host) holds desired_chans values, each in 0..255, or 0..65535 where the call's source elements are uint16 (native
 *   calls, index calls into uint16); NULL is all zeros.
 * View statuses in d_view_status [m], the first that applies: FPNGB_DECODE_BAD_VIEW when file is not in 0..n-1; the file's status
 *   when it is not 0; FPNGB_DECODE_BAD_CROP for an empty box or one not inside the image (the walk's test of the resized call);
 *   FPNGB_DECODE_BAD_VIEW for resize_h or resize_w outside 1..2^24, |offset_y| or |offset_x| above 2^24, or unknown flag bits;
 *   else 0.  The output image of a view whose status is not 0 is left untouched.
 * Files: every file is decoded, d_status [n] and d_info as in the ragged call; the walk checks no box (boxes belong to views), so
 *   FPNGB_DECODE_BAD_CROP is never a file status here.  pixel_cap, the bounds and the verify switch as in the resized call.
 * Call-level checks (a rejected call enqueues nothing and writes nothing): those of fpngb_decode_packed_resized_device, with the
 *   layout checked for m images, plus FPNGB_ERR_INVALID_ARG for m == 0 or m > 65535, a NULL d_views or d_view_status, and a fill
 *   value out of range.  n <= 65535 as there.
 * Stream-ordered, no host synchronisation: the launches of the resized call with the same flags (12, 14 with verify on, for an
 *   fpng-only call).  The resize or nearest kernel writes the view statuses itself and is profile slot 8. */
/* ---- bicubic resize in the resized and views decodes (opt-in: FPNGB_RESIZE_BICUBIC) ------------------------------------------
 * With flags & FPNGB_RESIZE_BICUBIC, fpngb_decode_packed_resized_device and fpngb_decode_packed_views_device resample by torch's
 * bicubic rule (F.interpolate(mode="bicubic", align_corners=False, antialias=...), torchvision's InterpolationMode.BICUBIC) in
 * place of the bilinear one.  Per axis, crop length `in`, output length `out`, output index i, every operation a separately
 * rounded fp32 one, scale = (float)in / (float)out as above:
 *   With FPNGB_RESIZE_ANTIALIAS (torch's _upsample_bicubic2d_aa), at EVERY scale, upscaling included (unlike bilinear, where the
 *   two rules coincide below scale 1 and aa needs scale >= 1):
 *     support  = scale >= 1 ? 2 * scale : 2;   invscale = scale >= 1 ? 1 / scale : 1
 *     center, xmin, xsize: the bilinear formulas above with this support
 *     w_j      = cubic(-0.5)((j + xmin - center + 0.5f) * invscale), j < xsize; then w_j /= sum(w) if the sum != 0
 *     cubic(a)(x) = ((a+2)|x| - (a+3)) x^2 + 1 for |x| < 1;  ((a|x| - 5a)|x| + 8a)|x| - 4a for 1 <= |x| < 2;  0 otherwise
 *   Without it (torch's upsample_bicubic2d):
 *     real = scale * (i + 0.5f) - 0.5f (not clamped at 0);  x0 = floorf(real);  t = real - x0
 *     taps x0 - 1, x0, x0 + 1, x0 + 2, each clamped to [0, in - 1] (the border of the CROP is replicated: torch interpolates the
 *     cropped tensor, so a tap left of `left` reads column `left`), weights, not normalised, with A = -0.75:
 *       cc2(t + 1), cc1(t), cc1(1 - t), cc2(2 - t);   cc1(x) = ((A+2)x - (A+3))x^2 + 1,   cc2(x) = ((Ax - 5A)x + 8A)x - 4A
 *   At identity size both give the weights (0, 1, 0, 0) exactly: the output is the source, bit for bit.
 *   Bicubic overshoots (values below 0 and above 255 on the 0-255 scale); r is stored by the rules above: uint8 cvt.rni.sat.u8(r)
 *   (torchvision v2's GPU uint8 path: float interpolate, clamp, round); float T(r * scale + bias) on the unclamped r; native calls
 *   cvt.rni.sat.u16(r), round_u8(r / 257) or T((r / 257) * scale + bias).
 * FPNGB_RESIZE_BICUBIC goes with FPNGB_RESIZE_ANTIALIAS, _ANY_PNG, _ALL_PNG_FORMATS, _NATIVE and views; with FPNGB_RESIZE_NEAREST,
 *   _NEAREST_EXACT or _INDEX it gives FPNGB_ERR_INVALID_ARG (bicubic on class ids is refused, as bilinear is).  Statuses, the fill,
 *   flips, placement, launches (12, 14 with verify on, for an fpng-only call), profile slot 8 and stream ordering are the bilinear
 *   call's. */
enum { FPNGB_RESIZE_BICUBIC = 256 };

enum { FPNGB_VIEW_HFLIP = 1, FPNGB_VIEW_VFLIP = 2 };
enum { FPNGB_DECODE_BAD_VIEW = 106 };   /* views decode only: a view row names no file of the call, or a bad size, offset or flag */
FPNGB_API int fpngb_decode_packed_views_device(const void* d_base, size_t base_bytes, const uint64_t* d_offsets, const uint32_t* d_sizes,
                                               uint32_t n, uint32_t max_file_size, uint32_t max_w, uint32_t max_h, size_t pixel_cap,
                                               const int32_t* d_views /* m x 10, device */, uint32_t m,
                                               uint32_t out_w, uint32_t out_h, uint32_t desired_chans, uint32_t flags,
                                               const fpngb_pixel_format* fmt /* NULL = uint8 */,
                                               const uint32_t* fill /* host, desired_chans values, or NULL */,
                                               void* d_out, size_t out_image_stride, size_t out_row_pitch, size_t out_pixel_stride,
                                               size_t out_chan_stride, uint32_t* d_info /* n*6 or NULL */, int32_t* d_status,
                                               int32_t* d_view_status, void* stream);

/* ---- typed encode input: float32 / float16 / bfloat16 pixels with a per-channel scale and bias, rounded to 8 bits ------------
 * The *_typed encode calls take the input as elements x of T (fmt->dtype: float32, float16 or bfloat16) and encode, for channel c,
 * the uint8 value
 *     f = (float)x                                        exact for all three types
 *     y = (f * scale[c]) + bias[c]                        two separately rounded fp32 operations, never an FMA
 *     q = NaN(y) ? 0 : clamp(round_half_to_even(y), 0, 255)
 *   so +-inf and out-of-range values saturate to 255 or 0.  In torch: torch.nan_to_num(x.float() * s + b, nan=0.0).round()
 *   .clamp(0, 255).to(torch.uint8).  The written file is byte-identical to what fpngb_encode_batch_device writes for the uint8
 *   image q, for every flag.  Rounding is half to even only; torchvision's save_image adds 0.5 and truncates, which differs on
 *   exact ties (x.5) alone.  Here scale and bias act on the input: the inverse of a typed decode's normalisation is
 *   scale = max_value * std, bias = max_value * mean.  Entries at an index >= the image's channel count are ignored.
 *   How: one conversion kernel reads the input once and writes tight uint8 rows into a library-owned device buffer of
 *   sum(w*h*chans) bytes (grow-only, kept between calls); the uint8 pipeline then encodes that buffer.  Each call adds that one
 *   launch to the uint8 call's, and fpngb_profile_read reports the conversion kernel in slot 9.
 * Call-level checks, in addition to the uint8 twin's (a rejected call enqueues nothing and writes nothing):
 *   FPNGB_ERR_INVALID_ARG for a NULL fmt, a dtype other than the three above, or a scale or bias entry in use (index < chans; for
 *   the ragged call, < the largest chans of the call) that is not finite;
 *   FPNGB_ERR_ALIGNMENT unless the pixel address(es) and every stride are multiples of sizeof(T);
 *   FPNGB_ERR_INVALID_ARG unless the strides divided by sizeof(T) form an interleaved or planar layout of "Pixel layouts" (pixel
 *   stride chans * sizeof(T), channel stride sizeof(T); or pixel stride sizeof(T)), size-1 dimensions canonicalised.  Inputs may
 *   overlap (stride 0 included).  All input addressing is 64-bit: no row-pitch limit, and one image's input may pass 4 GiB.
 * fpngb_encode_batch_device_typed: the arguments of fpngb_encode_batch_device_strided plus fmt; strides in BYTES.
 * fpngb_encode_ragged_device_typed: the arguments of fpngb_encode_ragged_device plus fmt; strides (or NULL for tight HWC rows of
 *   T) in BYTES.  One launch converts every image of the call (its descriptors go up with the call's other tables through the
 *   pinned staging ring).  Slots, d_out_offsets, d_sizes, fallbacks, stream ordering with no host synchronisation: the uint8 call's. */
FPNGB_API int fpngb_encode_batch_device_typed(const void* d_pixels, size_t image_stride, size_t row_pitch, size_t pixel_stride,
                                              size_t chan_stride, uint32_t n, uint32_t w, uint32_t h, uint32_t chans,
                                              const fpngb_pixel_format* fmt, uint32_t flags, void* d_out, size_t out_stride,
                                              uint32_t* d_sizes, void* stream);
FPNGB_API int fpngb_encode_ragged_device_typed(uint32_t n, const uint64_t* pixels, const uint32_t* dims, const uint64_t* strides,
                                               const fpngb_pixel_format* fmt, uint32_t flags, void* d_out, size_t out_cap,
                                               uint64_t* d_out_offsets, uint32_t* d_sizes, void* stream);

/* ---- typed PNG encode input: float32 / float16 / bfloat16 pixels to 8- or 16-bit PNG samples -------------------------------
 * fpngb_encode_png_ragged_device_typed: the arguments of fpngb_encode_png_ragged_device plus fmt.  Image i has an output depth
 * D_i (dims[4i + 3]: 8 or 16; the element type is fmt->dtype) and M = 2^D_i - 1.  Channel c of each element x of T becomes the
 * sample
 *     f = (float)x                                        exact for all three types
 *     y = (f * scale[c]) + bias[c]                        two separately rounded fp32 operations, never an FMA
 *     q = NaN(y) ? 0 : clamp(round_half_to_even(y), 0, M) cvt.rni.sat.u8.f32 / cvt.rni.sat.u16.f32
 *   For D = 8 this is the rule of the typed encode calls above, bit for bit.  Scale and bias are in the OUTPUT's units: depth in
 *   metres at D = 16 with scale 1000 writes millimetres.  In torch: torch.nan_to_num(x.float() * s + b, nan=0.0).round()
 *   .clamp(0, M).to(torch.uint8 or torch.uint16).
 *   The file written for image i is byte-identical, for every flag, to what fpngb_encode_png_ragged_device writes for the
 *   quantised uint8 / uint16 image q: D = 8 with 3 or 4 channels gives an fpng file (identical to fpngb_encode_ragged_device_typed's,
 *   fallbacks included), everything else the PNG format of DESIGN.md §4.6.
 *   Inverse of the native float decode: a 16-bit sample s decoded to float32 with scale k is x = fl(fl(s / 257) * k); encoding x
 *   at D = 16 with scale 257 / k gives s back, for every s (checked exhaustively for k = 257, 0.257 and 257 / 65535).  float16
 *   and bfloat16 cannot hold every 16-bit sample, so a lossless 16-bit round trip needs float32.
 *     strides  in BYTES of T (or NULL for tight HWC rows of T), the layouts of "Pixel layouts"; all input addressing is 64-bit,
 *              so the input rows have no 32-bit pitch limit.
 *   Slots, d_out_offsets, d_sizes, flags and stream ordering: those of fpngb_encode_png_ragged_device (slot i is sized by
 *   fpngb_max_encoded_size(w, h, chans * D_i / 8)).
 *   Call-level checks (a rejected call enqueues nothing and writes nothing): those of fpngb_encode_png_ragged_device, with its
 *   16-bit parity rule replaced by FPNGB_ERR_ALIGNMENT unless every address and stride is a multiple of sizeof(T); and
 *   FPNGB_ERR_INVALID_ARG for a NULL fmt, a dtype other than float32, float16 or bfloat16 (FPNGB_DTYPE_UINT16 input is the
 *   untyped call's), or a scale or bias entry in use (index < the call's largest chans) that is not finite.
 *   How: one conversion launch for the whole call, whatever its mix of depths, channel counts and layouts, writes tight rows of
 *   each image's samples (native little-endian uint16 for D = 16) into the library-owned buffer of the typed encode calls, which
 *   needs sum(align16(w * h * chans * D / 8)) bytes; then the untyped call's launches run on those rows.  fpngb_profile_read
 *   reports the conversion kernel in slot 9. */
FPNGB_API int fpngb_encode_png_ragged_device_typed(uint32_t n, const uint64_t* pixels, const uint32_t* dims, const uint64_t* strides,
                                                   const fpngb_pixel_format* fmt, uint32_t flags, void* d_out, size_t out_cap,
                                                   uint64_t* d_out_offsets, uint32_t* d_sizes, void* stream);

/* Pins the calling thread to the CPUs of the NUMA node of the library's GPU (sysfs: the GPU's PCI device -> numa_node ->
 * cpulist), so that pinned buffers allocated afterwards and the thread that issues the H2D/D2H copies are local to the GPU's
 * PCIe root port.  Call once per rank after fpngb_init(), before allocating staging memory.  Returns the node, or -1 if the
 * topology is not visible (nothing changed). */
FPNGB_API int fpngb_bind_host_thread_to_device_numa(void);

/* Pinned host memory helpers for callers that want full PCIe bandwidth through the *_host entry points. */
FPNGB_API void* fpngb_host_alloc(size_t bytes);
FPNGB_API void fpngb_host_free(void* p);

/* Number of kernels the library has launched since fpngb_init (bench.py reports it as gpu_launches). */
FPNGB_API uint64_t fpngb_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* FPNG_B200_H */
