// fpng_b200/csrc/container_kernels.cu -- container walk of files that are already in device memory.
//
// container_walk_kernel runs container_walk (container.cuh, the same function the host entry points use) with one thread
// per file: a file has a handful of chunks, and the only long loop is the CRC of an ancillary chunk, which one thread
// computes byte by byte from a 256-entry table in constant memory.
#include "container.cuh"
#include "decode.cuh"
#include "crc_math.cuh"

namespace fpngb {

struct CrcByteTable { uint32_t t[256]; };
static constexpr CrcByteTable make_crc_byte_table()
{
    CrcByteTable r{};
    for (uint32_t n = 0; n < 256; n++) {
        uint32_t c = n;
        for (int k = 0; k < 8; k++) c = (c & 1u) ? (kCrcPoly ^ (c >> 1)) : (c >> 1);
        r.t[n] = c;
    }
    return r;
}
__constant__ CrcByteTable c_walk_crc = make_crc_byte_table();

struct DeviceCrc {
    __device__ uint32_t operator()(const uint8_t* p, size_t n) const
    {
        uint32_t c = 0xFFFFFFFFu;
        for (size_t i = 0; i < n; i++) c = c_walk_crc.t[(c ^ p[i]) & 0xFFu] ^ (c >> 8);
        return ~c;
    }
};

__global__ void __launch_bounds__(128) container_walk_kernel(WalkParams p)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n) return;
    const unsigned long long ofs = p.offsets[i];
    const uint32_t size = p.sizes[i];
    uint32_t st, w = 0, h = 0, c = 0, io = 0, il = 0;
    if (!size) st = FPNGB_DECODE_INVALID_ARG;                                            // fpng.cpp:3092-3096
    else st = container_walk(p.base + ofs, size, DeviceCrc{}, &w, &h, &c, &io, &il);
    if (p.info) {
        uint32_t* o = p.info + (size_t)i * 6;
        o[0] = st; o[1] = w; o[2] = h; o[3] = c; o[4] = io; o[5] = il;
    }
    if (p.files) {
        // argument checks first, then the walk's code, then the call's shape
        uint32_t pre = st;
        if (!size || size > p.max_file_size || (ofs & 3ull)) pre = FPNGB_DECODE_INVALID_ARG;
        else if (!pre && (w != p.w || h != p.h || c != p.chans)) pre = FPNGB_DECODE_SHAPE_MISMATCH;
        FileDesc fd;
        fd.base = ofs; fd.file_size = size; fd.idat_ofs = pre ? 0u : io; fd.idat_len = pre ? 0u : il; fd.pre_status = pre;
        p.files[i] = fd;
    }
}

void launch_container_walk(const WalkParams& p, cudaStream_t s)
{
    container_walk_kernel<<<(p.n + 127) / 128, 128, 0, s>>>(p);
}

}  // namespace fpngb
