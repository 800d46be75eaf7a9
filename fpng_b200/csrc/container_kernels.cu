// fpng_b200/csrc/container_kernels.cu -- container walk of files that are already in device memory.
//
// container_walk_kernel runs container_walk (container.cuh, the same function the host entry points use) with one thread
// per file: a file has a handful of chunks, and the only long loop is the CRC of an ancillary chunk, which one thread
// computes byte by byte from a 256-entry table in constant memory.
#include "container.cuh"
#include "png_walk.cuh"
#include "decode.cuh"
#include "crc_math.cuh"

namespace fpngb {

__constant__ CrcByteTable c_walk_crc = crc_byte_table();

struct DeviceCrc {
    __device__ uint32_t operator()(const uint8_t* p, size_t n) const
    {
        uint32_t c = 0xFFFFFFFFu;
        for (size_t i = 0; i < n; i++) c = c_walk_crc.t[(c ^ p[i]) & 0xFFu] ^ (c >> 8);
        return ~c;
    }
};

// kAny (the any-PNG calls): files container_walk rejects with FPNGB_DECODE_NOT_FPNG are walked again by png_walk (with `flags`); a
// general file that passes every check of the call gets pre_status kPngPending (kPngPendingExt for the files png_walk marks ext)
// and, with png != nullptr, its PngDesc (decode.cuh).  A native call (FPNGB_PNG_NATIVE, with kAny) may pass desired 0: the
// w * h * desired check then uses the file's own channel count.  An index call (WalkParams::index, with FPNGB_PNG_ALL_FORMATS in
// flags, so fm describes every general file) gives FPNGB_DECODE_NOT_INDEXED right after the walk.
template <bool kAny>
__global__ void __launch_bounds__(128) container_walk_kernel(WalkParams p, PngDesc* png, uint32_t flags)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const unsigned long long ofs = p.offsets[i];
    const uint32_t size = p.sizes[i];
    const bool ragged = p.files && !p.chans;
    // argument checks: size 0 (fpng.cpp:3092-3096), and for the packed decodes the workspace bound and the alignment of the
    // decode kernels' word reads; the ragged call also keeps every file inside the buffer and walks only files that pass
    const bool bad_arg = !size || (p.files && (size > p.max_file_size || (ofs & 3ull) || (ragged && (ofs > p.base_bytes || size > p.base_bytes - ofs))));
    uint32_t st, w = 0, h = 0, c = 0, io = 0, il = 0;
    bool general = false;
    PngFormat fm{};
    if (!size || (ragged && bad_arg)) st = FPNGB_DECODE_INVALID_ARG;
    else if (kAny) st = any_png_walk(p.base + ofs, size, DeviceCrc{}, flags, &w, &h, &c, &io, &il, &general, &fm);
    else st = container_walk(p.base + ofs, size, DeviceCrc{}, &w, &h, &c, &io, &il);
    if (p.info) {
        uint32_t* o = p.info + (size_t)i * 6;
        o[0] = st; o[1] = w; o[2] = h; o[3] = c; o[4] = io; o[5] = il;
    }
    if (p.files) {
        // argument checks first, then the walk's code, then the call's shape
        uint32_t pre = bad_arg ? (uint32_t)FPNGB_DECODE_INVALID_ARG : st;
        // an index call stores one raw sample per pixel: palette indices, and gray samples of every depth but 16 into uint8
        if (kAny && !pre && p.index && !(general && (fm.type == 3 || (fm.type == 0 && (fm.depth < 16 || p.index == 2)))))
            pre = FPNGB_DECODE_NOT_INDEXED;
        if (!pre && ragged) {
            if (w > p.w || h > p.h) pre = FPNGB_DECODE_SHAPE_MISMATCH;
            else if ((unsigned long long)w * h * (kAny && !p.desired ? c : p.desired) > 0xFFFFFFFFull)
                pre = FPNGB_DECODE_FAILED_DIMENSIONS_TOO_LARGE;                     // fpng.cpp:3103-3105
            else if (p.boxes) {                                                     // the resized call's crop box
                const int32_t* b = p.boxes + (size_t)i * 4;
                const long long top = b[0], left = b[1], bh = b[2], bw = b[3];
                if (bh < 1 || bw < 1 || top < 0 || left < 0 || top + bh > h || left + bw > w) pre = FPNGB_DECODE_BAD_CROP;
            }
        } else if (!pre && (w != p.w || h != p.h || c != p.chans)) pre = FPNGB_DECODE_SHAPE_MISMATCH;
        if (kAny && !pre && general) pre = kPngPending;
        if (kAny && png) {
            const bool ok = pre == kPngPending, ext = ok && fm.ext;
            png[i] = ext ? PngDesc{0ull, il, 0u, fm.raw_len, fm.depth, fm.type, fm.interlace, fm.plte_ofs, fm.plte_n, fm.trns_ofs,
                                   fm.trns_len, 0u}
                         : PngDesc{0ull, ok ? il : 0u, 0u};
        }
        if (kAny && pre == kPngPending) pre = 0;                                // placed as any file; marked again below
        FileDesc fd;
        fd.base = ofs; fd.file_size = size; fd.idat_ofs = pre ? 0u : io; fd.idat_len = pre ? 0u : il; fd.pre_status = pre;
        if (ragged) {
            fd.w = w; fd.h = h; fd.chans = c; fd.pitch = delta_pitch(w, c);
            fd.delta_base = 0; fd.out_base = 0; fd.sub_base = 0;                 // decode_place_kernel
        } else {
            fd.w = p.w; fd.h = p.h; fd.chans = p.chans; fd.pitch = delta_pitch(p.w, p.chans);
            fd.delta_base = (unsigned long long)i * fd.pitch * p.h; fd.out_base = i * p.out_stride;
            fd.sub_base = (unsigned long long)i * subs_for(p.max_file_size);
        }
        if (kAny && general && !pre) fd.pre_status = fm.ext ? kPngPendingExt : kPngPending;
        p.files[i] = fd;
    }
}

void launch_container_walk(const WalkParams& p, cudaStream_t s)
{
    container_walk_kernel<false><<<(p.n + 127) / 128, 128, 0, s>>>(p, nullptr, 0u);
}
void launch_container_walk_any(const WalkParams& p, PngDesc* png, uint32_t flags, cudaStream_t s)
{
    container_walk_kernel<true><<<(p.n + 127) / 128, 128, 0, s>>>(p, png, flags);
}

// One CTA: exclusive scans of the output bytes, delta bytes and records of the accepted files, kPlaceThreads files per round.
// kAny: general files (pre_status kPngPending or kPngPendingExt) are placed too, with their inflated rows in the delta bytes (an
// ext file's PngDesc::raw_len), no records, and a fourth scan of their gathered zlib bytes (z_cap).  A native call (with kAny) may
// pass px_bytes 0: every file then takes chans * elem output bytes per pixel.
constexpr uint32_t kPlaceThreads = 1024;
template <bool kAny>
__global__ void __launch_bounds__(kPlaceThreads) decode_place_kernel(PlaceParams p, PngDesc* png, unsigned long long z_cap)
{
    constexpr int K = kAny ? 4 : 3;
    __shared__ unsigned long long s_warp[K][kPlaceThreads / 32];
    __shared__ unsigned long long s_carry[K];
    const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
    if (tid < K) s_carry[tid] = 0;
    for (uint32_t first = 0; first < p.n; first += kPlaceThreads) {
        const uint32_t i = first + tid;
        FileDesc fd{};
        bool placed = false, general = false;
        if (i < p.n) { fd = p.files[i]; general = kAny && png_pending(fd.pre_status); placed = fd.pre_status == 0 || general; }
        unsigned long long v[K];
#pragma unroll
        for (int k = 0; k < K; k++) v[k] = 0ull;
        if (placed) {
            const uint32_t px_bytes = kAny && !p.px_bytes ? fd.chans * p.elem : p.px_bytes;
            v[0] = ((unsigned long long)fd.w * fd.h * px_bytes + 15ull) & ~15ull;
            if (general) {
                const unsigned long long raw = fd.pre_status == kPngPendingExt ? png[i].raw_len
                                                                               : (unsigned long long)fd.h * (1ull + (unsigned long long)fd.w * fd.chans);
                v[1] = (raw + 15ull) & ~15ull;
                v[K - 1] = ((unsigned long long)png[i].zlen + 15ull) & ~15ull;
            } else {
                v[1] = (unsigned long long)fd.h * fd.pitch;
                v[2] = subs_for(fd.file_size);
            }
        }
        unsigned long long x[K];
#pragma unroll
        for (int k = 0; k < K; k++) {                      // inclusive warp scan, then the warp totals
            x[k] = v[k];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const unsigned long long u = __shfl_up_sync(0xFFFFFFFFu, x[k], o); if (lane >= (uint32_t)o) x[k] += u; }
            if (lane == 31) s_warp[k][warp] = x[k];
        }
        __syncthreads();
        if (warp == 0) {                                   // exclusive scan of the warp totals, carry of the earlier rounds in front
#pragma unroll
            for (int k = 0; k < K; k++) {
                unsigned long long t = s_warp[k][lane];
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const unsigned long long u = __shfl_up_sync(0xFFFFFFFFu, t, o); if (lane >= (uint32_t)o) t += u; }
                s_warp[k][lane] = s_carry[k] + t - s_warp[k][lane];
            }
        }
        __syncthreads();
        unsigned long long at[K];
#pragma unroll
        for (int k = 0; k < K; k++) at[k] = s_warp[k][warp] + x[k] - v[k];
        if (i < p.n) {
            p.out_offsets[i] = at[0];
            if (placed) {
                FileDesc* d = p.files + i;
                if (at[0] + v[0] > p.out_cap || at[1] + v[1] > p.delta_cap || at[2] + v[2] > p.sub_cap ||
                    (kAny && at[K - 1] + v[K - 1] > z_cap))
                    d->pre_status = FPNGB_DECODE_OUT_OF_SPACE;
                else {
                    d->out_base = at[0]; d->delta_base = at[1]; d->sub_base = at[2];
                    if (general) png[i].zofs = at[K - 1];
                }
            }
        }
        if (tid == kPlaceThreads - 1) for (int k = 0; k < K; k++) s_carry[k] = at[k] + v[k];
        __syncthreads();
    }
    if (tid == 0) p.out_offsets[p.n] = s_carry[0] | (s_carry[0] > p.out_cap ? 1ull << 63 : 0ull);
}

void launch_decode_place(const PlaceParams& p, cudaStream_t s)
{
    decode_place_kernel<false><<<1, kPlaceThreads, 0, s>>>(p, nullptr, 0ull);
}
void launch_decode_place_any(const PlaceParams& p, PngDesc* png, unsigned long long z_cap, cudaStream_t s)
{
    decode_place_kernel<true><<<1, kPlaceThreads, 0, s>>>(p, png, z_cap);
}

}  // namespace fpngb
