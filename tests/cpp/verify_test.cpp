// tests/cpp/verify_test.cpp -- a C++ caller of the drop-in API (namespace fpng) with the decoder's integrity check on
// (fpngb_set_decode_verify) and a general-PNG fallback registered: damaged files come back as FPNG_DECODE_FAILED_HEADER_CRC32 /
// FPNGB_DECODE_ADLER_MISMATCH and never reach the fallback, while a clean file still decodes.
#include "fpng.h"
#include "fpng_b200.h"

#include <stdio.h>
#include <stdlib.h>
#include <vector>

static int g_fallback_calls = 0;
static int fallback(const void*, uint32_t, uint32_t desired, void*, void** px, uint32_t* w, uint32_t* h, uint32_t* c)
{
    g_fallback_calls++;
    *px = malloc(desired); *w = 1; *h = 1; *c = desired;
    return 0;
}

static uint32_t be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }
static void put_be32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }

int main()
{
    fpng::fpng_init();
    fpngb_set_fallback_decoder(fallback, nullptr);
    if (fpngb_set_decode_verify(1) != 0 || fpngb_get_decode_verify() != 1) { printf("switch\n1 failures\n"); return 1; }
    const uint32_t w = 97, h = 23;
    std::vector<uint8_t> img(w * h * 3);
    for (size_t i = 0; i < img.size(); i++) img[i] = (uint8_t)((i * 7) / 5 + (i % 3) * 40);
    std::vector<uint8_t> png;
    if (!fpng::fpng_encode_image_to_memory(img.data(), w, h, 3, png, 0)) { printf("encode\n1 failures\n"); return 1; }
    uint32_t W, H, C, io = 0, il = 0;
    if (fpngb_get_info_ex(png.data(), (uint32_t)png.size(), &W, &H, &C, &io, &il) != 0) { printf("info\n1 failures\n"); return 1; }
    int failures = 0;
    std::vector<uint8_t> out;
    // clean file: decodes
    int st = fpng::fpng_decode_memory(png.data(), (uint32_t)png.size(), out, W, H, C, 3);
    if (st != 0 || out != img) { printf("clean file: status %d\n", st); failures++; }
    // Adler-32 rewritten, IDAT CRC recomputed: FPNGB_DECODE_ADLER_MISMATCH
    std::vector<uint8_t> a = png;
    a[io + 8 + il - 1] ^= 1;
    put_be32(&a[io + 8 + il], fpng::fpng_crc32(&a[io + 4], il + 4, 0));
    st = fpng::fpng_decode_memory(a.data(), (uint32_t)a.size(), out, W, H, C, 3);
    if (st != FPNGB_DECODE_ADLER_MISMATCH) { printf("adler: status %d\n", st); failures++; }
    // IDAT data byte changed, CRC left: FPNG_DECODE_FAILED_HEADER_CRC32
    std::vector<uint8_t> b = png;
    b[io + 8 + il / 2] ^= 0x10;
    if (be32(&b[io + 8 + il]) != be32(&png[io + 8 + il])) { printf("crc field moved\n"); failures++; }
    st = fpng::fpng_decode_memory(b.data(), (uint32_t)b.size(), out, W, H, C, 4);
    if (st != fpng::FPNG_DECODE_FAILED_HEADER_CRC32) { printf("crc: status %d\n", st); failures++; }
    if (g_fallback_calls) { printf("fallback called %d times\n", g_fallback_calls); failures++; }
    // with the switch off the file with the rewritten Adler-32 decodes as the reference decodes it
    fpngb_set_decode_verify(0);
    st = fpng::fpng_decode_memory(a.data(), (uint32_t)a.size(), out, W, H, C, 3);
    if (st != 0 || out != img) { printf("switch off, adler: status %d\n", st); failures++; }
    printf("%d failures\n", failures);
    return failures ? 1 : 0;
}
