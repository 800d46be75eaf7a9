// fpng_b200/csrc/fpng_dropin.cu -- namespace fpng wrappers (include/fpng.h) over the C ABI (include/fpng_b200.h).
// Ownership and error behaviour follow the reference (src/fpng.cpp:1662-1829, 3079-3190): the callee resizes the
// caller's vector, encode returns false on invalid arguments, decode zeroes its outputs first and maps every stream
// violation to FPNG_DECODE_NOT_FPNG.
#include "../../include/fpng.h"
#include "../../include/fpng_b200.h"

#include <stdio.h>
#include <stdlib.h>

#define DROPIN_API __attribute__((visibility("default")))

static fpngb_fallback_decoder g_fallback = nullptr;
static void* g_fallback_user = nullptr;
extern "C" {
void fpngb_set_fallback_decoder(fpngb_fallback_decoder fn, void* user) { g_fallback = fn; g_fallback_user = user; }
fpngb_fallback_decoder fpngb_get_fallback_decoder(void** user) { if (user) *user = g_fallback_user; return g_fallback; }
}

namespace fpng
{
    DROPIN_API void fpng_init()
    {
        int dev = -1;
        if (const char* e = getenv("FPNG_B200_DEVICE")) dev = atoi(e);
        const int rc = fpngb_init(dev);
        if (rc != FPNGB_OK) fprintf(stderr, "fpng_init: fpngb_init failed with code %d (no CUDA device? there is no CPU fallback)\n", rc);
    }

    DROPIN_API bool fpng_cpu_supports_sse41() { return false; }

    DROPIN_API uint32_t fpng_crc32(const void* pData, size_t size, uint32_t prev_crc32) { return fpngb_crc32(pData, size, prev_crc32); }
    DROPIN_API uint32_t fpng_adler32(const void* pData, size_t size, uint32_t adler) { return fpngb_adler32(pData, size, adler); }

    DROPIN_API bool fpng_encode_image_to_memory(const void* pImage, uint32_t w, uint32_t h, uint32_t num_chans, std::vector<uint8_t>& out_buf, uint32_t flags)
    {
        if (!pImage || w < 1 || h < 1 || (num_chans != 3 && num_chans != 4) || w > (1u << 24) || h > (1u << 24) || (uint64_t)w * h > 0xFFFFFFFFull)
            return false;
        const size_t cap = fpngb_max_encoded_size(w, h, num_chans);
        out_buf.resize(cap);
        size_t n = 0;
        const int rc = fpngb_encode_host(pImage, w, h, num_chans, flags, out_buf.data(), cap, &n);
        if (rc != FPNGB_OK) { out_buf.resize(0); return false; }
        out_buf.resize(n);
        return true;
    }

    DROPIN_API bool fpng_encode_image_to_file(const char* pFilename, const void* pImage, uint32_t w, uint32_t h, uint32_t num_chans, uint32_t flags)
    {
        std::vector<uint8_t> buf;
        if (!fpng_encode_image_to_memory(pImage, w, h, num_chans, buf, flags)) return false;
        FILE* f = fopen(pFilename, "wb");
        if (!f) return false;
        const bool ok = fwrite(buf.data(), 1, buf.size(), f) == buf.size();
        return (fclose(f) != EOF) && ok;
    }

    DROPIN_API int fpng_get_info(const void* pImage, uint32_t image_size, uint32_t& width, uint32_t& height, uint32_t& channels_in_file)
    {
        return fpngb_get_info(pImage, image_size, &width, &height, &channels_in_file);
    }

    // a registered general-PNG decoder takes over the files fpng rejects (fpngb_set_fallback_decoder, include/fpng_b200.h)
    static int try_fallback(const void* pImage, uint32_t image_size, std::vector<uint8_t>& out, uint32_t& width, uint32_t& height,
                            uint32_t& channels_in_file, uint32_t desired_channels)
    {
        if (!g_fallback) { out.resize(0); return FPNG_DECODE_NOT_FPNG; }
        void* px = nullptr; uint32_t w = 0, h = 0, c = 0;
        if (g_fallback(pImage, image_size, desired_channels, g_fallback_user, &px, &w, &h, &c) != 0 || !px) { out.resize(0); return FPNG_DECODE_NOT_FPNG; }
        out.assign((const uint8_t*)px, (const uint8_t*)px + (size_t)w * h * desired_channels);
        free(px);
        width = w; height = h; channels_in_file = c;
        return FPNG_DECODE_SUCCESS;
    }

    DROPIN_API int fpng_decode_memory(const void* pImage, uint32_t image_size, std::vector<uint8_t>& out, uint32_t& width, uint32_t& height,
                                      uint32_t& channels_in_file, uint32_t desired_channels)
    {
        out.resize(0);
        width = height = channels_in_file = 0;
        if (!pImage || !image_size || (desired_channels != 3 && desired_channels != 4)) return FPNG_DECODE_INVALID_ARG;
        int st = fpngb_get_info(pImage, image_size, &width, &height, &channels_in_file);
        if (st == FPNG_DECODE_NOT_FPNG) return try_fallback(pImage, image_size, out, width, height, channels_in_file, desired_channels);
        if (st) return st;
        const uint64_t need = (uint64_t)width * height * desired_channels;
        if (need > 0xFFFFFFFFull) return FPNG_DECODE_FAILED_DIMENSIONS_TOO_LARGE;
        out.resize((size_t)need);
        st = fpngb_decode_host(pImage, image_size, out.data(), out.size(), &width, &height, &channels_in_file, desired_channels);
        // a damaged file (fpngb_set_decode_verify: FPNG_DECODE_FAILED_HEADER_CRC32 / FPNGB_DECODE_ADLER_MISMATCH) is not handed to the fallback
        if (st == FPNG_DECODE_NOT_FPNG) return try_fallback(pImage, image_size, out, width, height, channels_in_file, desired_channels);
        return st;
    }

    DROPIN_API int fpng_decode_file(const char* pFilename, std::vector<uint8_t>& out, uint32_t& width, uint32_t& height,
                                    uint32_t& channels_in_file, uint32_t desired_channels)
    {
        FILE* f = fopen(pFilename, "rb");
        if (!f) return FPNG_DECODE_FILE_OPEN_FAILED;
        if (fseek(f, 0, SEEK_END) != 0) { fclose(f); return FPNG_DECODE_FILE_SEEK_FAILED; }
        const long long sz = ftello(f);
        if (fseek(f, 0, SEEK_SET) != 0) { fclose(f); return FPNG_DECODE_FILE_SEEK_FAILED; }
        if (sz < 0 || sz > 0xFFFFFFFFll) { fclose(f); return FPNG_DECODE_FILE_TOO_LARGE; }
        std::vector<uint8_t> buf((size_t)sz);
        if (fread(buf.data(), 1, buf.size(), f) != buf.size()) { fclose(f); return FPNG_DECODE_FILE_READ_FAILED; }
        fclose(f);
        return fpng_decode_memory(buf.data(), (uint32_t)buf.size(), out, width, height, channels_in_file, desired_channels);
    }
}
