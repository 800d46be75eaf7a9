// tests/cpp/layout_test.cpp -- the argument rules of fpng_b200/csrc/layout.h (check_layout, parse_format) on a CPU, for
// tests/test_layout_rules_cpu.py.  One case per input line, one answer per output line:
//   L mode base image row pixel chan n h w chans elem  ->  rc image row pixel chan planar
//     mode u8: a uint8 input under the uint8 encoder's 32-bit row-pitch limit; in: a typed input; out: an output
//   F null dtype chans scale0..3 bias0..3 (float bit patterns)  ->  rc dtype elem scale0..3 bias0..3 (bit patterns)
#include "../../fpng_b200/csrc/layout.h"
#include <stdio.h>
#include <string.h>

using namespace fpngb;

static unsigned bits(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
static float from_bits(unsigned u) { float f; memcpy(&f, &u, 4); return f; }

int main()
{
    char kind[4], mode[4];
    while (scanf("%3s", kind) == 1) {
        if (kind[0] == 'L') {
            unsigned long long base, image, row, pixel, chan;
            unsigned n, h, w, chans, elem;
            if (scanf("%3s %llu %llu %llu %llu %llu %u %u %u %u %u", mode, &base, &image, &row, &pixel, &chan, &n, &h, &w, &chans, &elem) != 11)
                return 2;
            Layout L{0, 0, 0, 0, false};
            int rc = check_layout((const void*)(uintptr_t)base, image, row, pixel, chan, n, h, w, chans, elem, strcmp(mode, "out") == 0, L);
            if (!rc && strcmp(mode, "u8") == 0 && L.row > 0xFFFFFFFFull) rc = FPNGB_ERR_INVALID_ARG;
            printf("%d %llu %llu %llu %llu %d\n", rc, (unsigned long long)L.image, (unsigned long long)L.row, (unsigned long long)L.pixel,
                   (unsigned long long)L.chan, L.planar ? 1 : 0);
        } else {
            unsigned null_fmt, dtype, chans, s[4], b[4];
            if (scanf("%u %u %u %x %x %x %x %x %x %x %x", &null_fmt, &dtype, &chans, &s[0], &s[1], &s[2], &s[3], &b[0], &b[1], &b[2], &b[3]) != 11)
                return 2;
            fpngb_pixel_format fmt;
            fmt.dtype = dtype;
            for (int c = 0; c < 4; c++) { fmt.scale[c] = from_bits(s[c]); fmt.bias[c] = from_bits(b[c]); }
            PixelFormat f = uint8_format();
            const int rc = parse_format(null_fmt ? nullptr : &fmt, chans, f);
            printf("%d %u %u", rc, f.dtype, f.elem);
            for (int c = 0; c < 4; c++) printf(" %x", bits(f.scale[c]));
            for (int c = 0; c < 4; c++) printf(" %x", bits(f.bias[c]));
            printf("\n");
        }
    }
    return 0;
}
