"""ctypes front-end for oracle/png_encode_oracle.c, the TEST-ONLY C restatement of the PNG files encode_png_device writes for
gray, gray+alpha and 16-bit images.  It is its own library, oracle/libpngenc_oracle.so: one translation unit with fpng_oracle.c
(which it includes for its Huffman helpers, bit writer and checksums), built by build() below.

Only tests/ and tools/ import this module.  The product package (fpng_b200) never does."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libpngenc_oracle.so")
SOURCES = [os.path.join(HERE, "png_encode_oracle.c"), os.path.join(HERE, "fpng_oracle.c")]


def build(force: bool = False) -> str:
    """Compile libpngenc_oracle.so when it is missing or older than its sources."""
    if force or not os.path.exists(SO) or any(os.path.getmtime(SO) < os.path.getmtime(s) for s in SOURCES):
        tmp = SO + ".building"
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-std=c11", "-fPIC", "-shared", "-Wall", "-Wextra", "-o", tmp,
                               SOURCES[0]], cwd=HERE)
        os.replace(tmp, SO)
    return SO


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class PngEncodeOracle:
    def __init__(self):
        L = C.CDLL(build())
        L.oracle_png_encode.restype = C.c_size_t
        L.oracle_png_encode.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p,
                                        C.c_size_t, C.c_void_p]
        L.oracle_max_encoded_size.restype = C.c_size_t
        L.oracle_max_encoded_size.argtypes = [C.c_uint32] * 3
        L.oracle_init()
        self.L = L

    def max_encoded_size(self, w, h, bytes_per_pixel) -> int:
        return self.L.oracle_max_encoded_size(w, h, bytes_per_pixel)

    def png_encode(self, img, flags=0, want_filters=False):
        """The file fpngb_encode_png_ragged_device writes for img, an [h, w, c] uint8 or uint16 array (c 1..4); with
        want_filters also the filter type of every row."""
        a = np.ascontiguousarray(img)
        assert a.ndim == 3 and a.dtype in (np.uint8, np.uint16), (a.shape, a.dtype)
        h, w, c = a.shape
        depth = 8 * a.dtype.itemsize
        cap = self.max_encoded_size(w, h, c * a.dtype.itemsize)
        out = np.empty(cap, dtype=np.uint8)
        filters = np.zeros(h, dtype=np.uint8)
        n = self.L.oracle_png_encode(_ptr(a), w, h, c, depth, flags, _ptr(out), cap, _ptr(filters))
        if n == 0:
            raise ValueError("oracle_png_encode rejected the arguments")
        data = out[:n].tobytes()
        return (data, filters) if want_filters else data
