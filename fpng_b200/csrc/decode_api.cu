// fpng_b200/csrc/decode_api.cu -- container walk (host) and decode entry points of the C ABI.
#include "../../include/fpng_b200.h"
#include "kernels.cuh"
#include "decode.cuh"
#include "container.cuh"
#include "png_walk.cuh"
#include "layout.h"
#include "runtime.h"
#include <string.h>
#include <atomic>
#include <vector>

namespace fpngb {

static Buffer g_dec_ws;        // FileDesc[n] | DecodeState[n] | luts | delta scratch

// fpngb_set_decode_verify: off at load; every decode call reads it once, under context().mu, when it enqueues
static std::atomic<int> g_decode_verify{0};

// Reserves the workspace of a decode call for n files, n_subs SubInfo records and delta_bytes of delta rows in all, orders it
// after the previous call's kernels, and points p's workspace fields into it (p.files included).  With verification on
// (fpngb_set_decode_verify), *verify points to n VerifyState records behind the rest; else it is nullptr.  extra_bytes more (the
// resized call's uint8 pixels and their offsets) go last, at *extra (256-byte aligned), and png_bytes more (the any-PNG calls'
// PngDesc records and gathered streams) behind them, at *png (256-byte aligned).  Caller holds context().mu.
static int decode_workspace_locked(uint32_t n, size_t n_subs, size_t delta_bytes, cudaStream_t s, DecodeParams& p, VerifyState** verify,
                                   size_t extra_bytes = 0, uint8_t** extra = nullptr, size_t png_bytes = 0, uint8_t** png = nullptr)
{
    size_t o = 0;
    const size_t o_files = o; o = align_up(o + (size_t)n * sizeof(FileDesc), 256);
    const size_t o_state = o; o = align_up(o + (size_t)n * sizeof(DecodeState), 256);
    const size_t o_luts = o; o = align_up(o + (size_t)n * 4096 * 4, 256);
    const size_t o_fast = o; o = align_up(o + (size_t)n * kFastWords * 4, 256);
    const size_t o_subs = o; o = align_up(o + n_subs * sizeof(SubInfo), 256);
    const size_t o_delta = o; o = align_up(o + delta_bytes + 64, 256);
    const bool verifying = g_decode_verify.load() != 0;
    const size_t o_verify = o; if (verifying) o = align_up(o + (size_t)n * sizeof(VerifyState), 256);
    const size_t o_extra = o; o += extra_bytes;
    const size_t o_png = png_bytes ? (o = align_up(o, 256)) : o; o += png_bytes;
    int rc = g_dec_ws.reserve(o); if (rc) return rc;
    rc = context().ws_acquire(s); if (rc) return rc;
    uint8_t* b = (uint8_t*)g_dec_ws.p;
    p.files = (const FileDesc*)(b + o_files); p.state = (DecodeState*)(b + o_state);
    p.luts = (uint32_t*)(b + o_luts); p.fast = (uint32_t*)(b + o_fast); p.subs = (SubInfo*)(b + o_subs);
    p.delta = b + o_delta;
    *verify = verifying ? (VerifyState*)(b + o_verify) : nullptr;
    if (extra) *extra = b + o_extra;
    if (png) *png = b + o_png;
    return 0;
}
// The same for n files of one shape whose IDAT chunks are at most max_idat bytes: file i's records and delta rows at i times the
// per-file share (the bases the uniform calls put in FileDesc), and the launch grids of that shape.
static int decode_workspace_uniform_locked(uint32_t n, uint32_t w, uint32_t h, uint32_t chans, uint32_t max_idat, cudaStream_t s,
                                           DecodeParams& p, VerifyState** verify)
{
    const int rc = decode_workspace_locked(n, (size_t)n * subs_for(max_idat), (size_t)n * delta_pitch(w, chans) * h, s, p, verify);
    if (rc) return rc;
    p.max_w = w; p.max_h = h; p.max_subs = subs_for(max_idat); p.chans = chans;
    return 0;
}

// Output layout of a decode call (layout.h): pixel (i, y, x, c) at d_out + i*image + y*row + x*pixel + c*chan.
static OutStrides set_output(DecodeParams& p, uint8_t* d_out, const Layout& L)
{
    p.d_out = d_out;
    return OutStrides{L.row, L.pixel, L.chan};
}

// Call-level checks shared by the device decode entry points: counts, channels and the container's shape limits
// (fpng.cpp:2966-2971: keeps w * chans and the scratch pitch inside 32 bits).
static int decode_shape_check(uint32_t w, uint32_t h, uint32_t chans_in_file, uint32_t desired_chans)
{
    if ((chans_in_file != 3 && chans_in_file != 4) || (desired_chans != 3 && desired_chans != 4) || !w || !h) return FPNGB_ERR_INVALID_ARG;
    if (w > (1u << 24) || h > (1u << 24) || (uint64_t)w * h > (1ull << 30)) return FPNGB_ERR_INVALID_ARG;
    if ((uint64_t)w * h * desired_chans > 0xFFFFFFFFull) return FPNGB_ERR_BUFFER_TOO_SMALL;
    return FPNGB_OK;
}
// The output format of a device decode call as the decode kernels take it: uint8 (typed false, fmt unused) or the *_typed call's
// fmt, checked over every channel the call may write (4 for a native call's desired 0).  A native call (FPNGB_PNG_NATIVE) also takes
// FPNGB_DTYPE_UINT16, whose scale and bias it ignores, as uint8 takes none.  elem receives the bytes per element.
static int decode_format(bool typed, const fpngb_pixel_format* fmt, uint32_t desired, bool native, TypedOut& t, uint32_t& elem)
{
    PixelFormat f = uint8_format();
    if (typed && native && fmt && fmt->dtype == FPNGB_DTYPE_UINT16) { f.dtype = FPNGB_DTYPE_UINT16; f.elem = 2; }
    else if (typed) { const int rc = parse_format(fmt, desired ? desired : 4, f); if (rc) return rc; }
    t = TypedOut{f.dtype, {}};
    memcpy(t.aff.scale, f.scale, sizeof f.scale); memcpy(t.aff.bias, f.bias, sizeof f.bias);
    elem = f.elem;
    return FPNGB_OK;
}

// Enqueue the decode pipeline for n files already resident on the device, file i at d_files + i * file_stride, described by host
// FileDescs (their base and pre_status are set here).  Caller holds context().mu.
static int decode_batch_locked(const uint8_t* d_files, size_t file_stride, const FileDesc* h_files, uint32_t n, uint32_t w, uint32_t h,
                               uint32_t chans, uint32_t desired, uint8_t* d_out, const Layout& out, uint32_t* d_status, cudaStream_t s,
                               const TypedOut* typed = nullptr)
{
    uint32_t max_idat = 0;
    for (uint32_t i = 0; i < n; i++) if (h_files[i].idat_len > max_idat) max_idat = h_files[i].idat_len;
    DecodeParams p{};
    VerifyState* verify = nullptr;
    int rc = decode_workspace_uniform_locked(n, w, h, chans, max_idat, s, p, &verify); if (rc) return rc;
    StageSlot* sl = nullptr;
    rc = context().stage_slot((size_t)n * sizeof(FileDesc), &sl); if (rc) return rc;
    FileDesc* staging = (FileDesc*)sl->buf.p;
    for (uint32_t i = 0; i < n; i++) {
        FileDesc& fd = staging[i];
        fd = h_files[i]; fd.base = (unsigned long long)i * file_stride; fd.pre_status = 0;
        fd.w = w; fd.h = h; fd.chans = chans; fd.pitch = delta_pitch(w, chans);
        fd.delta_base = (unsigned long long)i * fd.pitch * h; fd.out_base = (unsigned long long)i * out.image; fd.sub_base = (unsigned long long)i * p.max_subs;
    }
    FPNGB_CUDA_OK(cudaMemcpyAsync((void*)p.files, staging, (size_t)n * sizeof(FileDesc), cudaMemcpyHostToDevice, s));
    FPNGB_CUDA_OK(cudaEventRecord(sl->ev, s));
    p.d_files = d_files; p.d_status = d_status;
    // the CRC kernel's message ("IDAT" + stream) plus its misalignment stays within max_idat + 8 bytes
    launch_decode(p, set_output(p, d_out, out), n, desired, s, verify, (size_t)max_idat + 8, typed);
    count_launch(verify ? 10 : 8);
    FPNGB_CUDA_OK(cudaGetLastError());
    return context().ws_release(s);
}

// A device status of a file the host walked: FPNG_DECODE_NOT_FPNG for every stream violation (fpng.cpp:3131-3136), and the
// verify kernels' FPNG_DECODE_FAILED_HEADER_CRC32 / FPNGB_DECODE_ADLER_MISMATCH as they are.
static int host_status(uint32_t s)
{
    if (s == FPNGB_DECODE_FAILED_HEADER_CRC32 || s == FPNGB_DECODE_ADLER_MISMATCH) return (int)s;
    return s ? FPNGB_DECODE_NOT_FPNG : FPNGB_DECODE_SUCCESS;
}

// the host instantiation of the container walk (container.cuh)
struct HostCrc {
    uint32_t operator()(const uint8_t* p, size_t n) const { return host_crc32(p, n, 0); }
};
int container_info(const uint8_t* f, uint32_t size, uint32_t* w, uint32_t* h, uint32_t* chans, uint32_t* idat_ofs, uint32_t* idat_len)
{
    return container_walk(f, size, HostCrc{}, w, h, chans, idat_ofs, idat_len);
}

// The bodies of the device decode entry points: typed false is the uint8 call (fmt unused), true the *_typed one.
static int decode_batch_device_impl(const void* d_files, size_t file_stride, const uint32_t* file_sizes, const uint32_t* idat_ofs,
                                    const uint32_t* idat_len, uint32_t n, uint32_t w, uint32_t h, uint32_t chans_in_file,
                                    uint32_t desired_chans, void* d_out, size_t out_image_stride, size_t out_row_pitch,
                                    size_t out_pixel_stride, size_t out_chan_stride, bool typed, const fpngb_pixel_format* fmt,
                                    uint32_t* d_status, void* stream)
{
    Context& c = context();
    if (!c.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!d_files || !file_sizes || !idat_ofs || !idat_len || !d_out || !d_status || n == 0 || n > 65535) return FPNGB_ERR_INVALID_ARG;
    int rc = decode_shape_check(w, h, chans_in_file, desired_chans); if (rc) return rc;
    TypedOut t;
    uint32_t elem;
    rc = decode_format(typed, fmt, desired_chans, false, t, elem); if (rc) return rc;
    Layout out;
    rc = check_layout(d_out, out_image_stride, out_row_pitch, out_pixel_stride, out_chan_stride, n, h, w, desired_chans, elem, true, out);
    if (rc) return rc;
    if (file_stride % 4 || (uintptr_t)d_files % 4) return FPNGB_ERR_ALIGNMENT;
    std::vector<FileDesc> fds(n);
    for (uint32_t i = 0; i < n; i++) {
        if ((uint64_t)idat_ofs[i] + 8 + idat_len[i] + 4 > file_sizes[i] || file_sizes[i] > file_stride) return FPNGB_ERR_INVALID_ARG;
        fds[i] = FileDesc{}; fds[i].file_size = file_sizes[i]; fds[i].idat_ofs = idat_ofs[i]; fds[i].idat_len = idat_len[i];
    }
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    return decode_batch_locked((const uint8_t*)d_files, file_stride, fds.data(), n, w, h, chans_in_file, desired_chans, (uint8_t*)d_out,
                               out, d_status, (cudaStream_t)stream, typed ? &t : nullptr);
}

static int decode_packed_device_impl(const void* d_base, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n, uint32_t max_file_size,
                                     uint32_t w, uint32_t h, uint32_t chans_in_file, uint32_t desired_chans, void* d_out,
                                     size_t out_image_stride, size_t out_row_pitch, size_t out_pixel_stride, size_t out_chan_stride,
                                     bool typed, const fpngb_pixel_format* fmt, int32_t* d_status, void* stream)
{
    Context& c = context();
    if (!c.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!d_base || !d_offsets || !d_sizes || !d_out || !d_status || n == 0 || n > 65535 || !max_file_size) return FPNGB_ERR_INVALID_ARG;
    int rc = decode_shape_check(w, h, chans_in_file, desired_chans); if (rc) return rc;
    TypedOut t;
    uint32_t elem;
    rc = decode_format(typed, fmt, desired_chans, false, t, elem); if (rc) return rc;
    Layout out;
    rc = check_layout(d_out, out_image_stride, out_row_pitch, out_pixel_stride, out_chan_stride, n, h, w, desired_chans, elem, true, out);
    if (rc) return rc;
    if ((uintptr_t)d_base % 4) return FPNGB_ERR_ALIGNMENT;
    const cudaStream_t s = (cudaStream_t)stream;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    // an IDAT chunk is shorter than its file: max_file_size bounds the stream of every file that reaches the decode kernels
    DecodeParams p{};
    VerifyState* verify = nullptr;
    rc = decode_workspace_uniform_locked(n, w, h, chans_in_file, max_file_size, s, p, &verify); if (rc) return rc;
    WalkParams wp{};
    wp.base = (const uint8_t*)d_base; wp.offsets = (const unsigned long long*)d_offsets; wp.sizes = d_sizes; wp.n = n;
    wp.files = (FileDesc*)p.files; wp.max_file_size = max_file_size; wp.w = w; wp.h = h; wp.chans = chans_in_file;
    wp.out_stride = out.image;
    launch_container_walk(wp, s);
    p.d_files = (const uint8_t*)d_base; p.d_status = (uint32_t*)d_status;
    launch_decode(p, set_output(p, (uint8_t*)d_out, out), n, desired_chans, s, verify, max_file_size, typed ? &t : nullptr);
    count_launch(verify ? 11 : 9);
    FPNGB_CUDA_OK(cudaGetLastError());
    return context().ws_release(s);
}

// Workspace of the ragged call, from call arguments only (no host synchronisation).  Only files decode_place_kernel places and
// that fit in out_cap are decoded; they are a prefix of the placed files, so for every one of them the sums below run over
// decoded files alone.
//   records:   subs_for(s) <= s/128 + 3 per file of s bytes; files that lie inside the buffer and do not overlap have sizes that
//              sum to at most base_bytes, so base_bytes/128 + 3n records hold them all.  Every file also has s <= max_file_size.
//   delta:     a file needs h * align_up(w*c, 16) <= (4/desired) * (w*h*desired) + 15h bytes, h <= max_h and h <= w*h, and the
//              w*h*desired of the decoded files sum to at most out_cap.  Every file also needs at most max_h * pitch(max_w, 4).
//   any-PNG calls: a general file's inflated rows take align_up(h * (1 + w*c), 16) <= 4*w*h + 16h delta bytes (c <= 4, h >= 1), inside
//              the same bound from out_cap; from the shape, h * (delta_pitch(w, 4) + 16) per file.  Its gathered stream takes
//              align_up(zlen, 16) bytes, zlen < its size: at most base_bytes + 16n for files that do not overlap, and
//              align_up(max_file_size, 16) each.
//   all formats (FPNGB_PNG_ALL_FORMATS): an ext file of b <= 64 bits per pixel inflates to the rows of its passes, each of
//              1 + ceil(pw*b/8) bytes.  For b >= 8 the data bytes of all rows sum to w*h*b/8 <= 8wh; for b < 8 a row holds at most
//              pw bytes, so at most wh in all.  One filter byte per pass row: interlace 0 has h rows; Adam7's seven passes have
//              ceil(h/8) + ceil(h/8) + ceil((h-4)/8) + ceil(h/4) + ceil((h-2)/4) + ceil(h/2) + ceil((h-1)/2) <= 15h/8 + 6 rows, the
//              "2h + 6" Adam7 adds.  So align_up(raw_len, 16) <= 8wh + 2h + 21 <= 8wh + 32h (h >= 1): the bound from out_cap is
//              out_cap*8/desired + 32 * min(rows, rows_px), and from the shape h * (8w + 32) per file.  Both also bound the 8-bit
//              general and fpng files (4wh + 16h, and h * (delta_pitch(w, 4) + 16) <= h * (8w + 32)).  Flag off: the bounds above.
//   native (FPNGB_PNG_NATIVE): file i writes w*h*c_i values, c_i = desired, or its own channel count for desired 0, so c_i >= 1 and
//              the w*h*c_i of the decoded files sum to at most out_cap.  Every delta need above is a bound per pixel plus one per
//              row, so it holds with c_i := 1: an fpng file's h * align_up(w*c, 16) <= 4wh + 16h <= 4 (w*h*c_i) + 16h, a general
//              8-bit file's 4wh + 16h the same, an ext file's 8wh + 32h <= 8 (w*h*c_i) + 32h (the worst ratio: an RGBA16 file decoded
//              to 1 channel inflates up to 8 bytes per output value), and sum h <= sum w*h*c_i <= out_cap.  So the bounds above
//              hold with desired := 1; the bound from the shape does not depend on desired.
// A file whose range still ends past a bound (overlapping files) gets FPNGB_DECODE_OUT_OF_SPACE from decode_place_kernel.
static unsigned long long sat_u64(unsigned __int128 v) { return v > ~0ull ? ~0ull : (unsigned long long)v; }
static void ragged_workspace(uint32_t n, size_t base_bytes, uint32_t max_file_size, uint32_t max_w, uint32_t max_h, uint32_t desired,
                             size_t out_cap, bool any_png, bool all_formats, unsigned long long& sub_cap,
                             unsigned long long& delta_cap, unsigned long long& z_cap)
{
    typedef unsigned __int128 u128;
    const u128 by_bytes = (u128)base_bytes / 128 + 3 * (u128)n, by_max = (u128)n * subs_for(max_file_size);
    sub_cap = sat_u64(by_bytes < by_max ? by_bytes : by_max);
    const u128 rows = (u128)n * max_h, rows_px = ((u128)out_cap + desired - 1) / desired;
    const u128 px_bytes = all_formats ? 8 : 4, row_bytes = all_formats ? 32 : 16;
    const u128 by_out = ((u128)out_cap * px_bytes + desired - 1) / desired + row_bytes * (rows < rows_px ? rows : rows_px);
    const u128 by_shape = rows * (all_formats ? 8 * (u128)max_w + 32 : (u128)(delta_pitch(max_w, 4) + (any_png ? 16u : 0u)));
    delta_cap = sat_u64(by_out < by_shape ? by_out : by_shape);
    const u128 z_bytes = (u128)base_bytes + 16 * (u128)n, z_max = (u128)n * align_up((size_t)max_file_size, 16);
    z_cap = any_png ? sat_u64(z_bytes < z_max ? z_bytes : z_max) : 0ull;
}

// The resize step of fpngb_decode_packed_resized_device and fpngb_decode_packed_views_device: its checked output and arguments.
// views != nullptr (the views call): m output images from the view table, boxes unused.
struct ResizeOut {
    const int32_t* boxes; uint32_t out_w, out_h, flags;
    uint8_t* d_out; Layout out; TypedOut t;
    const int32_t* views; int32_t* view_status; uint32_t m; uint32_t fill[4];
};

// The ragged pipeline: walk, place, decode.  With rz (the resized call), the uint8 pixels and their offsets go to the decode
// workspace instead of d_out / d_out_offsets (both unused), out_cap is the call's pixel_cap, the walk checks rz->boxes (none in a
// views call: boxes belong to the views), and the resize kernel runs behind the decode, before the workspace is released.  any_png: the any-PNG walk and placement, and the
// general files' gather, inflate and unfilter kernels behind the fpng decode (decode.cuh, PngDesc); png_flags: png_walk's flags
// (FPNGB_PNG_ALL_FORMATS adds the ext files' unfilter kernel; FPNGB_PNG_NATIVE allows desired_chans 0..4 and the formats
// decode_format takes for a native call, typed exactly when fmt is given; FPNGB_PNG_INDEX, with both, the raw samples of desired 1
// into uint8 or uint16).
static int decode_packed_ragged_impl(const void* d_base, size_t base_bytes, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n,
                                     uint32_t max_file_size, uint32_t max_w, uint32_t max_h, uint32_t desired_chans, void* d_out,
                                     size_t out_cap, uint64_t* d_out_offsets, uint32_t* d_info, bool typed, const fpngb_pixel_format* fmt,
                                     int32_t* d_status, void* stream, const ResizeOut* rz = nullptr, bool any_png = false,
                                     uint32_t png_flags = 0)
{
    Context& c = context();
    if (!c.ready) return FPNGB_ERR_NOT_INITIALIZED;
    const bool native = any_png && (png_flags & FPNGB_PNG_NATIVE);
    if (!d_base || !d_offsets || !d_sizes || (!rz && (!d_out || !d_out_offsets)) || !d_status || n == 0 || n > 65535 || !max_file_size ||
        (native ? desired_chans > 4 || (rz && !desired_chans) : desired_chans != 3 && desired_chans != 4) || !max_w || !max_h ||
        max_w > (1u << 24) || max_h > (1u << 24))
        return FPNGB_ERR_INVALID_ARG;
    const bool index = any_png && (png_flags & FPNGB_PNG_INDEX);
    if (index && ((png_flags & (FPNGB_PNG_ALL_FORMATS | FPNGB_PNG_NATIVE)) != (FPNGB_PNG_ALL_FORMATS | FPNGB_PNG_NATIVE) ||
                  desired_chans != 1 || (typed && (!fmt || fmt->dtype != FPNGB_DTYPE_UINT16))))
        return FPNGB_ERR_INVALID_ARG;
    TypedOut t;
    uint32_t elem;
    int rc = decode_format(typed, fmt, desired_chans, native, t, elem); if (rc) return rc;
    if ((uintptr_t)d_base % 4 || (!rz && (uintptr_t)d_out % 16)) return FPNGB_ERR_ALIGNMENT;
    unsigned long long sub_cap = 0, delta_cap = 0, z_cap = 0;
    // the delta bound holds for out_cap in pixel values (w*h*desired of the decoded files sum to at most out_cap / elem)
    const bool all_formats = any_png && (png_flags & FPNGB_PNG_ALL_FORMATS);
    ragged_workspace(n, base_bytes, max_file_size, max_w, max_h, native ? 1u : desired_chans, out_cap / elem, any_png, all_formats, sub_cap,
                     delta_cap, z_cap);
    if (sub_cap > SIZE_MAX / sizeof(SubInfo) || delta_cap > SIZE_MAX / 2 || (rz && out_cap > SIZE_MAX / 2) || z_cap > SIZE_MAX / 4)
        return FPNGB_ERR_BUFFER_TOO_SMALL;
    const size_t png_desc_bytes = any_png ? align_up((size_t)n * sizeof(PngDesc), 256) : 0;
    const size_t offsets_bytes = align_up(((size_t)n + 1) * sizeof(uint64_t), 256);
    const cudaStream_t s = (cudaStream_t)stream;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    DecodeParams p{};
    VerifyState* verify = nullptr;
    uint8_t* extra = nullptr;
    uint8_t* png = nullptr;
    rc = decode_workspace_locked(n, sub_cap, delta_cap, s, p, &verify, rz ? offsets_bytes + out_cap : 0, &extra,
                                 any_png ? png_desc_bytes + z_cap : 0, &png);
    if (rc) return rc;
    if (rz) { d_out_offsets = (uint64_t*)extra; d_out = extra + offsets_bytes; }
    p.max_w = max_w; p.max_h = max_h; p.max_subs = subs_for(max_file_size); p.chans = 0;
    WalkParams wp{};
    wp.base = (const uint8_t*)d_base; wp.offsets = (const unsigned long long*)d_offsets; wp.sizes = d_sizes; wp.n = n; wp.info = d_info;
    wp.files = (FileDesc*)p.files; wp.max_file_size = max_file_size; wp.w = max_w; wp.h = max_h; wp.chans = 0; wp.desired = desired_chans;
    wp.base_bytes = base_bytes; wp.boxes = rz && !rz->views ? rz->boxes : nullptr; wp.index = index ? elem : 0u;
    if (any_png) launch_container_walk_any(wp, (PngDesc*)png, png_flags & FPNGB_PNG_ALL_FORMATS, s);
    else launch_container_walk(wp, s);
    PlaceParams pp{};
    pp.files = (FileDesc*)p.files; pp.n = n; pp.px_bytes = desired_chans * elem; pp.elem = elem;
    pp.out_cap = out_cap; pp.delta_cap = delta_cap; pp.sub_cap = sub_cap; pp.out_offsets = (unsigned long long*)d_out_offsets;
    if (any_png) launch_decode_place_any(pp, (PngDesc*)png, z_cap, s);
    else launch_decode_place(pp, s);
    p.d_files = (const uint8_t*)d_base; p.d_status = (uint32_t*)d_status; p.d_out = (uint8_t*)d_out;
    const TypedOut* tp = typed || native ? &t : nullptr;
    launch_decode(p, OutStrides{0, desired_chans * elem, elem}, n, desired_chans, s, verify, max_file_size, tp);
    if (any_png) {                                  // behind decode_status_kernel: the general files' final statuses
        PngParams q{};
        q.d_files = (const uint8_t*)d_base; q.files = p.files; q.png = (PngDesc*)png; q.z = png + png_desc_bytes; q.rows = p.delta;
        q.d_out = (uint8_t*)d_out; q.d_status = (uint32_t*)d_status; q.n = n; q.desired = desired_chans; q.verify = verify != nullptr;
        q.index = index;
        launch_png_decode(q, tp, png_flags, s);
    }
    if (rz) {
        ResizeParams rp{};
        rp.px = (const uint8_t*)d_out; rp.px_offsets = (const unsigned long long*)d_out_offsets; rp.files = p.files; rp.d_status = d_status;
        rp.boxes = rz->boxes; rp.d_out = rz->d_out;
        rp.image = rz->out.image; rp.row = rz->out.row; rp.pixel = rz->out.pixel; rp.chan = rz->out.chan;
        rp.out_w = rz->out_w; rp.out_h = rz->out_h; rp.antialias = rz->flags & FPNGB_RESIZE_ANTIALIAS;
        rp.nearest = (rz->flags & FPNGB_RESIZE_NEAREST) ? 1u : (rz->flags & FPNGB_RESIZE_NEAREST_EXACT) ? 2u : 0u;
        rp.views = rz->views; rp.view_status = rz->view_status; rp.n = n; memcpy(rp.fill, rz->fill, sizeof rp.fill);
        decode_profile_mark_resize(s, false);
        launch_decode_resize(rp, rz->t, t.dtype, rz->views ? rz->m : n, desired_chans, (rz->flags & FPNGB_RESIZE_BICUBIC) != 0, s);
        decode_profile_mark_resize(s, true);
    }
    count_launch((verify ? 13 : 11) + (rz ? 1 : 0) + (any_png ? 3 : 0) + (all_formats ? 1 : 0));
    FPNGB_CUDA_OK(cudaGetLastError());
    return context().ws_release(s);
}

}  // namespace fpngb

using namespace fpngb;

extern "C" {

int fpngb_decode_batch_device_strided(const void* d_files, size_t file_stride, const uint32_t* file_sizes, const uint32_t* idat_ofs,
                                      const uint32_t* idat_len, uint32_t n, uint32_t w, uint32_t h, uint32_t chans_in_file,
                                      uint32_t desired_chans, void* d_out, size_t out_image_stride, size_t out_row_pitch,
                                      size_t out_pixel_stride, size_t out_chan_stride, uint32_t* d_status, void* stream)
{
    return decode_batch_device_impl(d_files, file_stride, file_sizes, idat_ofs, idat_len, n, w, h, chans_in_file, desired_chans, d_out,
                                    out_image_stride, out_row_pitch, out_pixel_stride, out_chan_stride, false, nullptr, d_status, stream);
}

int fpngb_decode_batch_device_typed(const void* d_files, size_t file_stride, const uint32_t* file_sizes, const uint32_t* idat_ofs,
                                    const uint32_t* idat_len, uint32_t n, uint32_t w, uint32_t h, uint32_t chans_in_file,
                                    uint32_t desired_chans, void* d_out, size_t out_image_stride, size_t out_row_pitch,
                                    size_t out_pixel_stride, size_t out_chan_stride, const fpngb_pixel_format* fmt, uint32_t* d_status,
                                    void* stream)
{
    return decode_batch_device_impl(d_files, file_stride, file_sizes, idat_ofs, idat_len, n, w, h, chans_in_file, desired_chans, d_out,
                                    out_image_stride, out_row_pitch, out_pixel_stride, out_chan_stride, true, fmt, d_status, stream);
}

int fpngb_decode_batch_device(const void* d_files, size_t file_stride, const uint32_t* file_sizes, const uint32_t* idat_ofs,
                              const uint32_t* idat_len, uint32_t n, uint32_t w, uint32_t h, uint32_t chans_in_file,
                              uint32_t desired_chans, void* d_out, size_t out_stride, uint32_t* d_status, void* stream)
{
    if (!context().ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!d_files || !file_sizes || !idat_ofs || !idat_len || !d_out || !d_status || n == 0 || n > 65535) return FPNGB_ERR_INVALID_ARG;
    const int rc = decode_shape_check(w, h, chans_in_file, desired_chans); if (rc) return rc;
    if (out_stride < (size_t)w * h * desired_chans) return FPNGB_ERR_BUFFER_TOO_SMALL;
    return fpngb_decode_batch_device_strided(d_files, file_stride, file_sizes, idat_ofs, idat_len, n, w, h, chans_in_file, desired_chans, d_out,
                                             out_stride, (size_t)w * desired_chans, desired_chans, 1, d_status, stream);
}

int fpngb_decode_host(const void* file, uint32_t size, void* out, size_t out_cap, uint32_t* w, uint32_t* h, uint32_t* chans, uint32_t desired)
{
    uint32_t ww = 0, hh = 0, cc = 0, idat_ofs = 0, idat_len = 0;
    if (w) *w = 0; if (h) *h = 0; if (chans) *chans = 0;
    if (!file || !size || !out || (desired != 3 && desired != 4)) return FPNGB_DECODE_INVALID_ARG;     // fpng.cpp:3092-3096
    const int st = container_info((const uint8_t*)file, size, &ww, &hh, &cc, &idat_ofs, &idat_len);
    if (w) *w = ww; if (h) *h = hh; if (chans) *chans = cc;
    if (st) return st;
    const uint64_t need = (uint64_t)ww * hh * desired;
    if (need > 0xFFFFFFFFull) return FPNGB_DECODE_FAILED_DIMENSIONS_TOO_LARGE;                          // fpng.cpp:3103-3105
    if (out_cap < need) return FPNGB_DECODE_INVALID_ARG;
    Context& c = context();
    if (!c.ready) return FPNGB_DECODE_INVALID_ARG;
    std::lock_guard<std::mutex> lk(c.mu);
    if (cudaSetDevice(c.device) != cudaSuccess) return FPNGB_DECODE_INVALID_ARG;
    const size_t fstride = align_up((size_t)size + 16, 16);
    if (c.dev_in.reserve(fstride) || c.dev_out.reserve(align_up(need, 16) + 64)) return FPNGB_DECODE_INVALID_ARG;
    uint32_t* d_status = (uint32_t*)((uint8_t*)c.dev_out.p + align_up(need, 16));
    cudaStream_t s = c.stream;
    cudaMemcpyAsync(c.dev_in.p, file, size, cudaMemcpyHostToDevice, s);
    FileDesc fd{}; fd.file_size = size; fd.idat_ofs = idat_ofs; fd.idat_len = idat_len;
    if (decode_batch_locked((const uint8_t*)c.dev_in.p, fstride, &fd, 1, ww, hh, cc, desired, (uint8_t*)c.dev_out.p,
                            tight_layout(ww, desired, align_up(need, 16)), d_status, s))
        return FPNGB_DECODE_INVALID_ARG;
    uint32_t* h_status = (uint32_t*)c.pin_small.p;
    cudaMemcpyAsync(h_status, d_status, 4, cudaMemcpyDeviceToHost, s);
    if (cudaStreamSynchronize(s) != cudaSuccess) return FPNGB_DECODE_INVALID_ARG;
    if (*h_status) return host_status(*h_status);
    cudaMemcpyAsync(out, c.dev_out.p, need, cudaMemcpyDeviceToHost, s);
    if (cudaStreamSynchronize(s) != cudaSuccess) return FPNGB_DECODE_INVALID_ARG;
    return FPNGB_DECODE_SUCCESS;
}

int fpngb_get_info(const void* file, uint32_t size, uint32_t* w, uint32_t* h, uint32_t* chans)
{
    uint32_t a, b, ww = 0, hh = 0, cc = 0;
    if (!file) { if (w) *w = 0; if (h) *h = 0; if (chans) *chans = 0; return FPNGB_DECODE_INVALID_ARG; }
    const int st = container_info((const uint8_t*)file, size, &ww, &hh, &cc, &a, &b);
    if (w) *w = ww; if (h) *h = hh; if (chans) *chans = cc;
    return st;
}

// Pipelined host-buffer batch decode: per chunk the files go H2D, the decode kernels run, the pixels come back D2H;
// three slots keep copies and kernels of neighbouring chunks overlapped.  Files that fail the container walk keep their
// status and are skipped; all decodable files must share width/height/channels.
int fpngb_decode_batch_host(const void* const* files, const uint32_t* sizes, uint32_t n, uint32_t desired, void* out, size_t out_stride,
                            uint32_t* w_out, uint32_t* h_out, uint32_t* chans_out, int* status)
{
    Context& c = context();
    if (!c.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!files || !sizes || !out || !status || n == 0 || (desired != 3 && desired != 4)) return FPNGB_ERR_INVALID_ARG;
    std::vector<FileDesc> fds(n);
    uint32_t W = 0, H = 0, C = 0, max_size = 0;
    for (uint32_t i = 0; i < n; i++) {
        uint32_t ww = 0, hh = 0, cc = 0, io = 0, il = 0;
        status[i] = (!files[i] || !sizes[i]) ? FPNGB_DECODE_INVALID_ARG : container_info((const uint8_t*)files[i], sizes[i], &ww, &hh, &cc, &io, &il);
        fds[i] = FileDesc{}; fds[i].file_size = sizes[i]; fds[i].idat_ofs = io; fds[i].idat_len = il;
        if (status[i]) continue;
        if (!W) { W = ww; H = hh; C = cc; }
        else if (ww != W || hh != H || cc != C) return FPNGB_ERR_INVALID_ARG;
        if (sizes[i] > max_size) max_size = sizes[i];
    }
    if (w_out) *w_out = W; if (h_out) *h_out = H; if (chans_out) *chans_out = C;
    if (!W) return FPNGB_OK;                                   // nothing decodable: statuses say why
    const uint64_t need = (uint64_t)W * H * desired;
    if (need > 0xFFFFFFFFull) { for (uint32_t i = 0; i < n; i++) if (!status[i]) status[i] = FPNGB_DECODE_FAILED_DIMENSIONS_TOO_LARGE; return FPNGB_OK; }
    if (out_stride < need) return FPNGB_ERR_BUFFER_TOO_SMALL;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));

    constexpr int kSlots = 3;
    const size_t fstride = align_up((size_t)max_size + 16, 16), pstride = align_up((size_t)need, 16);
    uint32_t per_chunk = (uint32_t)(((size_t)64 << 20) / need); if (per_chunk < 1) per_chunk = 1; if (per_chunk > n) per_chunk = n;
    if (per_chunk > 65535u) per_chunk = 65535u;                     // grid.y limit of the batch kernels (tiny images)
    const size_t slot_in = per_chunk * fstride, slot_out = per_chunk * pstride + align_up(per_chunk * 4, 256);
    int rc = c.dev_in.reserve(kSlots * slot_in); if (rc) return rc;
    rc = c.dev_out.reserve(kSlots * slot_out); if (rc) return rc;
    rc = c.pin_small.reserve(kSlots * align_up(per_chunk * 4, 256)); if (rc) return rc;
    if (!c.copy_in) { FPNGB_CUDA_OK(cudaStreamCreateWithFlags(&c.copy_in, cudaStreamNonBlocking)); FPNGB_CUDA_OK(cudaStreamCreateWithFlags(&c.copy_out, cudaStreamNonBlocking)); }
    EventSet<3 * kSlots> evs;                                       // destroyed on every exit path
    if (!evs.ok) return FPNGB_ERR_INTERNAL;
    cudaEvent_t* ev_in = evs.ev; cudaEvent_t* ev_done = evs.ev + kSlots; cudaEvent_t* ev_out = evs.ev + 2 * kSlots;
    // decodable files, in order
    std::vector<uint32_t> idx; idx.reserve(n);
    for (uint32_t i = 0; i < n; i++) if (!status[i]) idx.push_back(i);
    const uint32_t m = (uint32_t)idx.size(), nchunks = (m + per_chunk - 1) / per_chunk;
    int result = FPNGB_OK;
    std::vector<FileDesc> cf(per_chunk);
    for (uint32_t k = 0; k < nchunks && result == FPNGB_OK; k++) {
        const int sl = k % kSlots;
        const uint32_t first = k * per_chunk, cnt = (first + per_chunk <= m) ? per_chunk : m - first;
        if (k >= kSlots) {   // the slot's previous pixels and statuses have left the device
            if (cudaEventSynchronize(ev_out[sl]) != cudaSuccess) { result = FPNGB_ERR_INTERNAL; break; }
            const uint32_t pf = (k - kSlots) * per_chunk, pc = (pf + per_chunk <= m) ? per_chunk : m - pf;
            const uint32_t* hs = (const uint32_t*)((uint8_t*)c.pin_small.p + sl * align_up(per_chunk * 4, 256));
            for (uint32_t j = 0; j < pc; j++) status[idx[pf + j]] = host_status(hs[j]);
        }
        uint8_t* din = (uint8_t*)c.dev_in.p + sl * slot_in;
        uint8_t* dout = (uint8_t*)c.dev_out.p + sl * slot_out;
        uint32_t* dst = (uint32_t*)(dout + per_chunk * pstride);
        for (uint32_t j = 0; j < cnt; j++) {
            const uint32_t i = idx[first + j];
            cudaMemcpyAsync(din + j * fstride, files[i], sizes[i], cudaMemcpyHostToDevice, c.copy_in);
            cf[j] = fds[i];
        }
        cudaEventRecord(ev_in[sl], c.copy_in);
        cudaStreamWaitEvent(c.stream, ev_in[sl], 0);
        rc = decode_batch_locked(din, fstride, cf.data(), cnt, W, H, C, desired, dout, tight_layout(W, desired, pstride), dst, c.stream);
        if (rc) { result = rc; break; }
        cudaEventRecord(ev_done[sl], c.stream);
        cudaStreamWaitEvent(c.copy_out, ev_done[sl], 0);
        cudaMemcpyAsync((uint8_t*)c.pin_small.p + sl * align_up(per_chunk * 4, 256), dst, cnt * 4, cudaMemcpyDeviceToHost, c.copy_out);
        for (uint32_t j = 0; j < cnt; j++)
            cudaMemcpyAsync((uint8_t*)out + (size_t)idx[first + j] * out_stride, dout + j * pstride, need, cudaMemcpyDeviceToHost, c.copy_out);
        cudaEventRecord(ev_out[sl], c.copy_out);
    }
    cudaStreamSynchronize(c.copy_in); cudaStreamSynchronize(c.stream); cudaStreamSynchronize(c.copy_out);
    if (result == FPNGB_OK) {
        for (uint32_t k = (nchunks > kSlots ? nchunks - kSlots : 0); k < nchunks; k++) {
            const int sl = k % kSlots;
            const uint32_t pf = k * per_chunk, pc = (pf + per_chunk <= m) ? per_chunk : m - pf;
            const uint32_t* hs = (const uint32_t*)((uint8_t*)c.pin_small.p + sl * align_up(per_chunk * 4, 256));
            for (uint32_t j = 0; j < pc; j++) status[idx[pf + j]] = host_status(hs[j]);
        }
        if (cudaGetLastError() != cudaSuccess) result = FPNGB_ERR_INTERNAL;
    }
    return result;
}

// per-kernel device times (ms) of the most recent decode call made while profiling was on: prepare, scan, link, write, stored, unfilter,
// and for a verified call IDAT CRC and Adler-32
FPNGB_API int fpngb_set_decode_verify(int on)
{
    std::lock_guard<std::mutex> lk(context().mu);        // a call in flight keeps the setting it read
    g_decode_verify.store(on != 0);
    return FPNGB_OK;
}
FPNGB_API int fpngb_get_decode_verify(void) { return g_decode_verify.load(); }

FPNGB_API int fpngb_decode_profile_enable(int on) { decode_profile_enable(on != 0); return 0; }
FPNGB_API int fpngb_decode_profile_read(float* ms, int n) { return decode_profile_read(ms, n); }
// test hook: number of subsequences the link pass had to decode again since the last reset (synchronises the device)
FPNGB_API unsigned long long fpngb_debug_decode_repairs(int reset) { cudaDeviceSynchronize(); return decode_link_repairs(reset != 0); }
// test hook: speculative lead-in (bits) of the scan kernel for later decode calls, default 256; 0 makes nearly every guessed subsequence
// start wrong, so the link pass has to repair it.  Pixels and statuses never depend on it.  FPNGB_ERR_INVALID_ARG (unchanged) above 256.
FPNGB_API int fpngb_debug_decode_preroll(uint32_t bits) { return decode_set_pre_roll(bits) ? FPNGB_OK : FPNGB_ERR_INVALID_ARG; }

int fpngb_get_info_ex(const void* file, uint32_t size, uint32_t* w, uint32_t* h, uint32_t* chans, uint32_t* idat_ofs, uint32_t* idat_len)
{
    if (!file || !w || !h || !chans || !idat_ofs || !idat_len) return FPNGB_DECODE_INVALID_ARG;
    return container_info((const uint8_t*)file, size, w, h, chans, idat_ofs, idat_len);
}

int fpngb_get_info_batch_device(const void* d_base, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n, uint32_t* d_info, void* stream)
{
    Context& c = context();
    if (!c.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!d_base || !d_offsets || !d_sizes || !d_info || n == 0) return FPNGB_ERR_INVALID_ARG;
    WalkParams p{};
    p.base = (const uint8_t*)d_base; p.offsets = (const unsigned long long*)d_offsets; p.sizes = d_sizes; p.n = n; p.info = d_info;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    launch_container_walk(p, (cudaStream_t)stream);
    count_launch(1);
    FPNGB_CUDA_OK(cudaGetLastError());
    return FPNGB_OK;
}


int fpngb_decode_packed_device_strided(const void* d_base, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n, uint32_t max_file_size,
                                       uint32_t w, uint32_t h, uint32_t chans_in_file, uint32_t desired_chans, void* d_out,
                                       size_t out_image_stride, size_t out_row_pitch, size_t out_pixel_stride, size_t out_chan_stride,
                                       int32_t* d_status, void* stream)
{
    return decode_packed_device_impl(d_base, d_offsets, d_sizes, n, max_file_size, w, h, chans_in_file, desired_chans, d_out, out_image_stride,
                                     out_row_pitch, out_pixel_stride, out_chan_stride, false, nullptr, d_status, stream);
}

int fpngb_decode_packed_device_typed(const void* d_base, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n, uint32_t max_file_size,
                                     uint32_t w, uint32_t h, uint32_t chans_in_file, uint32_t desired_chans, void* d_out,
                                     size_t out_image_stride, size_t out_row_pitch, size_t out_pixel_stride, size_t out_chan_stride,
                                     const fpngb_pixel_format* fmt, int32_t* d_status, void* stream)
{
    return decode_packed_device_impl(d_base, d_offsets, d_sizes, n, max_file_size, w, h, chans_in_file, desired_chans, d_out, out_image_stride,
                                     out_row_pitch, out_pixel_stride, out_chan_stride, true, fmt, d_status, stream);
}

int fpngb_decode_packed_device(const void* d_base, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n, uint32_t max_file_size,
                               uint32_t w, uint32_t h, uint32_t chans_in_file, uint32_t desired_chans, void* d_out, size_t out_stride,
                               int32_t* d_status, void* stream)
{
    if (!context().ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!d_base || !d_offsets || !d_sizes || !d_out || !d_status || n == 0 || n > 65535 || !max_file_size) return FPNGB_ERR_INVALID_ARG;
    const int rc = decode_shape_check(w, h, chans_in_file, desired_chans); if (rc) return rc;
    if (out_stride < (size_t)w * h * desired_chans) return FPNGB_ERR_BUFFER_TOO_SMALL;
    return fpngb_decode_packed_device_strided(d_base, d_offsets, d_sizes, n, max_file_size, w, h, chans_in_file, desired_chans, d_out, out_stride,
                                              (size_t)w * desired_chans, desired_chans, 1, d_status, stream);
}



int fpngb_decode_packed_ragged_device(const void* d_base, size_t base_bytes, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n,
                                      uint32_t max_file_size, uint32_t max_w, uint32_t max_h, uint32_t desired_chans, void* d_out,
                                      size_t out_cap, uint64_t* d_out_offsets, uint32_t* d_info, int32_t* d_status, void* stream)
{
    return decode_packed_ragged_impl(d_base, base_bytes, d_offsets, d_sizes, n, max_file_size, max_w, max_h, desired_chans, d_out, out_cap,
                                     d_out_offsets, d_info, false, nullptr, d_status, stream);
}

int fpngb_decode_packed_ragged_device_typed(const void* d_base, size_t base_bytes, const uint64_t* d_offsets, const uint32_t* d_sizes,
                                            uint32_t n, uint32_t max_file_size, uint32_t max_w, uint32_t max_h, uint32_t desired_chans,
                                            void* d_out, size_t out_cap, uint64_t* d_out_offsets, uint32_t* d_info,
                                            const fpngb_pixel_format* fmt, int32_t* d_status, void* stream)
{
    return decode_packed_ragged_impl(d_base, base_bytes, d_offsets, d_sizes, n, max_file_size, max_w, max_h, desired_chans, d_out, out_cap,
                                     d_out_offsets, d_info, true, fmt, d_status, stream);
}

}  // extern "C"

namespace fpngb {

// The body of fpngb_decode_packed_resized_device (views nullptr, m = n) and fpngb_decode_packed_views_device (m views, boxes
// unused): the call-level checks of both, then the ragged pipeline with the resize step.
static int decode_resized_impl(const void* d_base, size_t base_bytes, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n,
                               uint32_t max_file_size, uint32_t max_w, uint32_t max_h, size_t pixel_cap, const int32_t* d_boxes,
                               const int32_t* d_views, uint32_t m, uint32_t out_w, uint32_t out_h, uint32_t desired_chans, uint32_t flags,
                               const fpngb_pixel_format* fmt, const uint32_t* fill, void* d_out, size_t out_image_stride,
                               size_t out_row_pitch, size_t out_pixel_stride, size_t out_chan_stride, uint32_t* d_info, int32_t* d_status,
                               int32_t* d_view_status, void* stream)
{
    if (!context().ready) return FPNGB_ERR_NOT_INITIALIZED;
    const bool native = (flags & FPNGB_RESIZE_NATIVE) != 0, index = (flags & FPNGB_RESIZE_INDEX) != 0;
    const uint32_t nearest = flags & (FPNGB_RESIZE_NEAREST | FPNGB_RESIZE_NEAREST_EXACT);
    const uint32_t index_needs = FPNGB_RESIZE_ANY_PNG | FPNGB_RESIZE_ALL_PNG_FORMATS | FPNGB_RESIZE_NATIVE;
    if (!d_out || n == 0 || n > 65535 || m == 0 || m > 65535 || !out_w || !out_h || out_w > (1u << 24) || out_h > (1u << 24) ||
        (native ? desired_chans < 1 || desired_chans > 4 : desired_chans != 3 && desired_chans != 4) ||
        (flags & ~(uint32_t)(FPNGB_RESIZE_ANTIALIAS | FPNGB_RESIZE_ANY_PNG | FPNGB_RESIZE_ALL_PNG_FORMATS | FPNGB_RESIZE_NATIVE |
                             FPNGB_RESIZE_NEAREST | FPNGB_RESIZE_NEAREST_EXACT | FPNGB_RESIZE_INDEX | FPNGB_RESIZE_BICUBIC)) ||
        ((flags & (FPNGB_RESIZE_ALL_PNG_FORMATS | FPNGB_RESIZE_NATIVE)) && !(flags & FPNGB_RESIZE_ANY_PNG)) ||
        nearest == (FPNGB_RESIZE_NEAREST | FPNGB_RESIZE_NEAREST_EXACT) || (nearest && (flags & FPNGB_RESIZE_ANTIALIAS)) ||
        ((flags & FPNGB_RESIZE_BICUBIC) && (nearest || index)) ||
        (index && ((flags & index_needs) != index_needs || !nearest || desired_chans != 1 || (fmt && fmt->dtype != FPNGB_DTYPE_UINT16))))
        return FPNGB_ERR_INVALID_ARG;
    ResizeOut rz{};
    rz.boxes = d_boxes; rz.out_w = out_w; rz.out_h = out_h; rz.flags = flags; rz.d_out = (uint8_t*)d_out;
    rz.views = d_views; rz.view_status = d_view_status; rz.m = m;
    if (d_views) {                  // the fill: a source value, so 16 bits where the call's source elements are uint16
        if (!d_view_status) return FPNGB_ERR_INVALID_ARG;
        const uint32_t fill_max = native && (!index || (fmt && fmt->dtype == FPNGB_DTYPE_UINT16)) ? 0xFFFFu : 0xFFu;
        for (uint32_t c = 0; fill && c < desired_chans; c++) {
            if (fill[c] > fill_max) return FPNGB_ERR_INVALID_ARG;
            rz.fill[c] = fill[c];
        }
    }
    uint32_t elem;
    int rc = decode_format(fmt != nullptr, fmt, desired_chans, native, rz.t, elem); if (rc) return rc;
    rc = check_layout(d_out, out_image_stride, out_row_pitch, out_pixel_stride, out_chan_stride, m, out_h, out_w, desired_chans, elem, true,
                      rz.out);
    if (rc) return rc;
    // native: the ragged decode holds every file as uint16 values in the 16-bit domain (pixel_cap counts their bytes); index: as
    // raw samples of the output's element type
    static const fpngb_pixel_format u16 = {FPNGB_DTYPE_UINT16, {0, 0, 0, 0}, {0, 0, 0, 0}};
    const uint32_t png_flags = ((flags & FPNGB_RESIZE_ALL_PNG_FORMATS) ? (uint32_t)FPNGB_PNG_ALL_FORMATS : 0u) |
                               (native ? (uint32_t)FPNGB_PNG_NATIVE : 0u) | (index ? (uint32_t)FPNGB_PNG_INDEX : 0u);
    const fpngb_pixel_format* mid = index ? fmt : native ? &u16 : nullptr;
    return decode_packed_ragged_impl(d_base, base_bytes, d_offsets, d_sizes, n, max_file_size, max_w, max_h, desired_chans, nullptr, pixel_cap,
                                     nullptr, d_info, mid != nullptr, mid, d_status, stream, &rz, (flags & FPNGB_RESIZE_ANY_PNG) != 0,
                                     png_flags);
}

}  // namespace fpngb

extern "C" {

int fpngb_decode_packed_resized_device(const void* d_base, size_t base_bytes, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n,
                                       uint32_t max_file_size, uint32_t max_w, uint32_t max_h, size_t pixel_cap, const int32_t* d_boxes,
                                       uint32_t out_w, uint32_t out_h, uint32_t desired_chans, uint32_t flags, const fpngb_pixel_format* fmt,
                                       void* d_out, size_t out_image_stride, size_t out_row_pitch, size_t out_pixel_stride,
                                       size_t out_chan_stride, uint32_t* d_info, int32_t* d_status, void* stream)
{
    return decode_resized_impl(d_base, base_bytes, d_offsets, d_sizes, n, max_file_size, max_w, max_h, pixel_cap, d_boxes, nullptr, n, out_w,
                               out_h, desired_chans, flags, fmt, nullptr, d_out, out_image_stride, out_row_pitch, out_pixel_stride,
                               out_chan_stride, d_info, d_status, nullptr, stream);
}

int fpngb_decode_packed_views_device(const void* d_base, size_t base_bytes, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n,
                                     uint32_t max_file_size, uint32_t max_w, uint32_t max_h, size_t pixel_cap, const int32_t* d_views,
                                     uint32_t m, uint32_t out_w, uint32_t out_h, uint32_t desired_chans, uint32_t flags,
                                     const fpngb_pixel_format* fmt, const uint32_t* fill, void* d_out, size_t out_image_stride,
                                     size_t out_row_pitch, size_t out_pixel_stride, size_t out_chan_stride, uint32_t* d_info,
                                     int32_t* d_status, int32_t* d_view_status, void* stream)
{
    if (!d_views) return context().ready ? FPNGB_ERR_INVALID_ARG : FPNGB_ERR_NOT_INITIALIZED;
    return decode_resized_impl(d_base, base_bytes, d_offsets, d_sizes, n, max_file_size, max_w, max_h, pixel_cap, nullptr, d_views, m, out_w,
                               out_h, desired_chans, flags, fmt, fill, d_out, out_image_stride, out_row_pitch, out_pixel_stride,
                               out_chan_stride, d_info, d_status, d_view_status, stream);
}

int fpngb_decode_packed_png_device_ex(const void* d_base, size_t base_bytes, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n,
                                      uint32_t max_file_size, uint32_t max_w, uint32_t max_h, uint32_t desired_chans, void* d_out,
                                      size_t out_cap, uint64_t* d_out_offsets, uint32_t* d_info, uint32_t flags,
                                      const fpngb_pixel_format* fmt, int32_t* d_status, void* stream)
{
    if (flags & ~(uint32_t)(FPNGB_PNG_ALL_FORMATS | FPNGB_PNG_NATIVE | FPNGB_PNG_INDEX))
        return context().ready ? FPNGB_ERR_INVALID_ARG : FPNGB_ERR_NOT_INITIALIZED;
    return decode_packed_ragged_impl(d_base, base_bytes, d_offsets, d_sizes, n, max_file_size, max_w, max_h, desired_chans, d_out, out_cap,
                                     d_out_offsets, d_info, fmt != nullptr, fmt, d_status, stream, nullptr, true, flags);
}

int fpngb_decode_packed_png_device(const void* d_base, size_t base_bytes, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n,
                                   uint32_t max_file_size, uint32_t max_w, uint32_t max_h, uint32_t desired_chans, void* d_out,
                                   size_t out_cap, uint64_t* d_out_offsets, uint32_t* d_info, const fpngb_pixel_format* fmt,
                                   int32_t* d_status, void* stream)
{
    return fpngb_decode_packed_png_device_ex(d_base, base_bytes, d_offsets, d_sizes, n, max_file_size, max_w, max_h, desired_chans, d_out,
                                             out_cap, d_out_offsets, d_info, 0u, fmt, d_status, stream);
}

int fpngb_get_png_info_batch_device_ex(const void* d_base, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n, uint32_t flags,
                                       uint32_t* d_info, void* stream)
{
    Context& c = context();
    if (!c.ready) return FPNGB_ERR_NOT_INITIALIZED;
    if (!d_base || !d_offsets || !d_sizes || !d_info || n == 0 || (flags & ~(uint32_t)FPNGB_PNG_ALL_FORMATS)) return FPNGB_ERR_INVALID_ARG;
    WalkParams p{};
    p.base = (const uint8_t*)d_base; p.offsets = (const unsigned long long*)d_offsets; p.sizes = d_sizes; p.n = n; p.info = d_info;
    std::lock_guard<std::mutex> lk(c.mu);
    FPNGB_CUDA_OK(cudaSetDevice(c.device));
    launch_container_walk_any(p, nullptr, flags, (cudaStream_t)stream);
    count_launch(1);
    FPNGB_CUDA_OK(cudaGetLastError());
    return FPNGB_OK;
}

int fpngb_get_png_info_batch_device(const void* d_base, const uint64_t* d_offsets, const uint32_t* d_sizes, uint32_t n, uint32_t* d_info,
                                    void* stream)
{
    return fpngb_get_png_info_batch_device_ex(d_base, d_offsets, d_sizes, n, 0u, d_info, stream);
}

int fpngb_get_png_info_ex(const void* file, uint32_t size, uint32_t flags, uint32_t* w, uint32_t* h, uint32_t* chans, uint32_t* idat_ofs,
                          uint32_t* idat_len)
{
    if (!file || !w || !h || !chans || !idat_ofs || !idat_len || (flags & ~(uint32_t)FPNGB_PNG_ALL_FORMATS)) return FPNGB_DECODE_INVALID_ARG;
    bool general;
    PngFormat fm;
    return any_png_walk((const uint8_t*)file, size, HostCrc{}, flags, w, h, chans, idat_ofs, idat_len, &general, &fm);
}

int fpngb_get_png_info(const void* file, uint32_t size, uint32_t* w, uint32_t* h, uint32_t* chans, uint32_t* idat_ofs, uint32_t* idat_len)
{
    return fpngb_get_png_info_ex(file, size, 0u, w, h, chans, idat_ofs, idat_len);
}

uint64_t fpngb_debug_png_raw_len(uint32_t w, uint32_t h, uint32_t bits_per_pixel, uint32_t interlace)
{
    return png_raw_len(w, h, bits_per_pixel, interlace);
}

}  // extern "C"
