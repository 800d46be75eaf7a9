"""ctypes binding of the C ABI declared in include/fpng_b200.h.  Fails loudly when the CUDA library is missing:
there is no CPU fallback anywhere in this package."""
from __future__ import annotations

import ctypes as C
import os

from . import _build

_lib = None

u32p = C.POINTER(C.c_uint32)


class PixelFormat(C.Structure):
    """fpngb_pixel_format: the element type (FPNGB_DTYPE_*) and per-channel scale and bias of the *_typed decode and encode calls"""
    _fields_ = [("dtype", C.c_uint32), ("scale", C.c_float * 4), ("bias", C.c_float * 4)]


class LabelPalette(C.Structure):
    """fpngb_label_palette: entries x chans (3 or 4) colour bytes in host memory; entries 0 is a gray label map"""
    _fields_ = [("colors", C.c_void_p), ("entries", C.c_uint32), ("chans", C.c_uint32)]


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    variant = os.environ.get("FPNGB_LIB_VARIANT")            # developer A/B builds (_build.build_variant); must exist
    if variant:
        path = os.path.join(_build.PKG, "_variants", f"libfpng_b200_{variant}.so")
        if not os.path.exists(path):
            raise FileNotFoundError(path)
    if not os.path.exists(path):
        # On a dev box without the prebuilt .so: compile it (needs nvcc); never substitute another implementation.
        _build.build()
    L = C.CDLL(path)
    L.fpngb_init.restype = C.c_int
    L.fpngb_init.argtypes = [C.c_int]
    L.fpngb_is_initialized.restype = C.c_int
    L.fpngb_version.restype = C.c_char_p
    L.fpngb_max_encoded_size.restype = C.c_size_t
    L.fpngb_max_encoded_size.argtypes = [C.c_uint32] * 3
    L.fpngb_encode_host.restype = C.c_int
    L.fpngb_encode_host.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t,
                                    C.POINTER(C.c_size_t)]
    L.fpngb_encode_batch_device.restype = C.c_int
    L.fpngb_encode_batch_device.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                            C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.fpngb_encode_batch_device_strided.restype = C.c_int
    L.fpngb_encode_batch_device_strided.argtypes = [C.c_void_p] + [C.c_size_t] * 4 + [C.c_uint32] * 5 + [C.c_void_p, C.c_size_t, C.c_void_p,
                                                                                                      C.c_void_p]
    L.fpngb_encode_batch_host.restype = C.c_int
    L.fpngb_encode_batch_host.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                          C.c_void_p, C.c_size_t, C.c_void_p]
    L.fpngb_get_info.restype = C.c_int
    L.fpngb_get_info.argtypes = [C.c_void_p, C.c_uint32, u32p, u32p, u32p]
    L.fpngb_decode_host.restype = C.c_int
    L.fpngb_decode_host.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, u32p, u32p, u32p, C.c_uint32]
    L.fpngb_get_info_ex.restype = C.c_int
    L.fpngb_get_info_ex.argtypes = [C.c_void_p, C.c_uint32, u32p, u32p, u32p, u32p, u32p]
    L.fpngb_decode_batch_device.restype = C.c_int
    L.fpngb_decode_batch_device.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32,
                                            C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.fpngb_decode_batch_device_strided.restype = C.c_int
    L.fpngb_decode_batch_device_strided.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_uint32] * 5 + \
        [C.c_void_p] + [C.c_size_t] * 4 + [C.c_void_p, C.c_void_p]
    L.fpngb_get_info_batch_device.restype = C.c_int
    L.fpngb_get_info_batch_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p]
    L.fpngb_decode_packed_device.restype = C.c_int
    L.fpngb_decode_packed_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                             C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.fpngb_decode_packed_device_strided.restype = C.c_int
    L.fpngb_decode_packed_device_strided.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p] + [C.c_uint32] * 6 + [C.c_void_p] + \
        [C.c_size_t] * 4 + [C.c_void_p, C.c_void_p]
    L.fpngb_decode_packed_ragged_device.restype = C.c_int
    L.fpngb_decode_packed_ragged_device.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p] + [C.c_uint32] * 5 + \
        [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.fpngb_decode_batch_device_typed.restype = C.c_int
    L.fpngb_decode_batch_device_typed.argtypes = L.fpngb_decode_batch_device_strided.argtypes[:-2] + [C.POINTER(PixelFormat), C.c_void_p,
                                                                                                   C.c_void_p]
    L.fpngb_decode_packed_device_typed.restype = C.c_int
    L.fpngb_decode_packed_device_typed.argtypes = L.fpngb_decode_packed_device_strided.argtypes[:-2] + [C.POINTER(PixelFormat), C.c_void_p,
                                                                                                     C.c_void_p]
    L.fpngb_decode_packed_ragged_device_typed.restype = C.c_int
    L.fpngb_decode_packed_ragged_device_typed.argtypes = L.fpngb_decode_packed_ragged_device.argtypes[:-2] + [C.POINTER(PixelFormat),
                                                                                                           C.c_void_p, C.c_void_p]
    L.fpngb_decode_packed_png_device.restype = C.c_int
    L.fpngb_decode_packed_png_device.argtypes = L.fpngb_decode_packed_ragged_device_typed.argtypes
    L.fpngb_get_png_info_batch_device.restype = C.c_int
    L.fpngb_get_png_info_batch_device.argtypes = L.fpngb_get_info_batch_device.argtypes
    L.fpngb_get_png_info.restype = C.c_int
    L.fpngb_get_png_info.argtypes = L.fpngb_get_info_ex.argtypes
    L.fpngb_decode_packed_png_device_ex.restype = C.c_int
    L.fpngb_decode_packed_png_device_ex.argtypes = L.fpngb_decode_packed_ragged_device.argtypes[:-2] + [C.c_uint32, C.POINTER(PixelFormat),
                                                                                                     C.c_void_p, C.c_void_p]
    L.fpngb_get_png_info_batch_device_ex.restype = C.c_int
    L.fpngb_get_png_info_batch_device_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    L.fpngb_get_png_info_ex.restype = C.c_int
    L.fpngb_get_png_info_ex.argtypes = L.fpngb_get_info_ex.argtypes[:2] + [C.c_uint32] + L.fpngb_get_info_ex.argtypes[2:]
    L.fpngb_debug_png_raw_len.restype = C.c_uint64
    L.fpngb_debug_png_raw_len.argtypes = [C.c_uint32] * 4
    L.fpngb_decode_packed_resized_device.restype = C.c_int
    L.fpngb_decode_packed_resized_device.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p] + [C.c_uint32] * 4 + \
        [C.c_size_t, C.c_void_p] + [C.c_uint32] * 4 + [C.POINTER(PixelFormat), C.c_void_p] + [C.c_size_t] * 4 + [C.c_void_p] * 3
    L.fpngb_decode_packed_views_device.restype = C.c_int
    L.fpngb_decode_packed_views_device.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p] + [C.c_uint32] * 4 + \
        [C.c_size_t, C.c_void_p] + [C.c_uint32] * 5 + [C.POINTER(PixelFormat), C.POINTER(C.c_uint32), C.c_void_p] + [C.c_size_t] * 4 + \
        [C.c_void_p] * 4
    L.fpngb_encode_batch_device_typed.restype = C.c_int
    L.fpngb_encode_batch_device_typed.argtypes = [C.c_void_p] + [C.c_size_t] * 4 + [C.c_uint32] * 4 + [C.POINTER(PixelFormat), C.c_uint32,
                                                                                                   C.c_void_p, C.c_size_t, C.c_void_p,
                                                                                                   C.c_void_p]
    L.fpngb_encode_ragged_device_typed.restype = C.c_int
    L.fpngb_encode_ragged_device_typed.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(PixelFormat), C.c_uint32,
                                                   C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    L.fpngb_compact_batch_device.restype = C.c_int
    L.fpngb_compact_batch_device.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.fpngb_compact_packed_device.restype = C.c_int
    L.fpngb_compact_packed_device.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.fpngb_encode_ragged_device.restype = C.c_int
    L.fpngb_encode_ragged_device.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t,
                                             C.c_void_p, C.c_void_p, C.c_void_p]
    L.fpngb_encode_png_ragged_device.restype = C.c_int
    L.fpngb_encode_png_ragged_device.argtypes = L.fpngb_encode_ragged_device.argtypes
    L.fpngb_max_reduced_encoded_size.restype = C.c_size_t
    L.fpngb_max_reduced_encoded_size.argtypes = [C.c_uint32] * 4
    L.fpngb_max_label_encoded_size.restype = C.c_size_t
    L.fpngb_max_label_encoded_size.argtypes = [C.c_uint32] * 3 + [C.POINTER(LabelPalette)]
    L.fpngb_encode_label_ragged_device.restype = C.c_int
    L.fpngb_encode_label_ragged_device.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                                   C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    L.fpngb_encode_png_ragged_device_typed.restype = C.c_int
    L.fpngb_encode_png_ragged_device_typed.argtypes = L.fpngb_encode_ragged_device_typed.argtypes
    L.fpngb_decode_batch_host.restype = C.c_int
    L.fpngb_decode_batch_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_size_t, u32p, u32p, u32p, C.c_void_p]
    L.fpngb_train_accumulate_device.restype = C.c_int
    L.fpngb_train_accumulate_device.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
    L.fpngb_create_dynamic_block_prefix.restype = C.c_int
    L.fpngb_create_dynamic_block_prefix.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64),
                                                    C.POINTER(C.c_int), C.c_void_p, C.c_void_p]
    L.fpngb_set_static_table.restype = C.c_int
    L.fpngb_set_static_table.argtypes = [C.c_uint32, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32]
    L.fpngb_crc32.restype = C.c_uint32
    L.fpngb_crc32.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32]
    L.fpngb_adler32.restype = C.c_uint32
    L.fpngb_adler32.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32]
    L.fpngb_host_alloc.restype = C.c_void_p
    L.fpngb_host_alloc.argtypes = [C.c_size_t]
    L.fpngb_host_free.restype = None
    L.fpngb_host_free.argtypes = [C.c_void_p]
    L.fpngb_crc32_ex.restype = C.c_int
    L.fpngb_crc32_ex.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, u32p]
    L.fpngb_adler32_ex.restype = C.c_int
    L.fpngb_adler32_ex.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, u32p]
    L.fpngb_comm_unique_id.restype = C.c_int
    L.fpngb_comm_unique_id.argtypes = [C.c_void_p]
    L.fpngb_comm_init.restype = C.c_int
    L.fpngb_comm_init.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.fpngb_comm_adopt.restype = C.c_int
    L.fpngb_comm_adopt.argtypes = [C.c_void_p]
    L.fpngb_comm_destroy.restype = C.c_int
    L.fpngb_comm_info.restype = C.c_int
    L.fpngb_comm_info.argtypes = [C.POINTER(C.c_int)] * 3
    L.fpngb_gather_setup.restype = C.c_int
    L.fpngb_gather_setup.argtypes = [C.c_size_t, C.c_uint32]
    L.fpngb_gather_encoded_device.restype = C.c_int
    L.fpngb_gather_encoded_device.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint32, C.c_int, C.POINTER(C.c_void_p),
                                              C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.c_void_p]
    L.fpngb_set_decode_verify.restype = C.c_int
    L.fpngb_set_decode_verify.argtypes = [C.c_int]
    L.fpngb_get_decode_verify.restype = C.c_int
    L.fpngb_get_decode_verify.argtypes = []
    L.fpngb_bind_host_thread_to_device_numa.restype = C.c_int
    L.fpngb_launch_count.restype = C.c_uint64
    L.fpngb_debug_use_fused.restype = None
    L.fpngb_debug_use_fused.argtypes = [C.c_int]
    L.fpngb_debug_crc_overlap.restype = None
    L.fpngb_debug_crc_overlap.argtypes = [C.c_int]
    L.fpngb_debug_decode_repairs.restype = C.c_ulonglong
    L.fpngb_debug_decode_repairs.argtypes = [C.c_int]
    L.fpngb_debug_decode_preroll.restype = C.c_int
    L.fpngb_debug_decode_preroll.argtypes = [C.c_uint32]
    L.fpngb_debug_rows_per_warp.restype = None
    L.fpngb_debug_rows_per_warp.argtypes = [C.c_uint32]
    L.fpngb_debug_static_table.restype = C.c_int
    L.fpngb_debug_static_table.argtypes = [C.c_uint32, C.c_void_p, C.c_void_p, u32p]
    _lib = L
    return L


class FpngB200Error(RuntimeError):
    pass


_ERR = {1: "invalid argument", 2: "output buffer too small", 3: "fpng_init() has not been called",
        4: "no CUDA device (this package has no CPU fallback)", 5: "pointer/stride alignment", 6: "internal error"}


def _nccl_msg(rc: int) -> str:
    return f"NCCL error {rc - 2000}"


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = _ERR.get(rc, _nccl_msg(rc) if rc >= 2000 else (f"CUDA error {rc - 1000}" if rc >= 1000 else f"code {rc}"))
        raise FpngB200Error(f"{what}: {msg}")
