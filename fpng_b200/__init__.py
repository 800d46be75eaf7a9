"""fpng_b200 -- H100-native (sm_90a) implementation of fpng's 24/32bpp PNG encode/decode hot path.

Host-side mirror of the reference's public interface (src/fpng.h): same names, argument meaning and error behaviour,
backed by hand-written CUDA kernels through the C ABI in include/fpng_b200.h.  No CPU fallback.
"""
from .api import (  # noqa: F401
    FPNG_ENCODE_SLOWER, FPNG_FORCE_UNCOMPRESSED,
    FPNG_DECODE_SUCCESS, FPNG_DECODE_NOT_FPNG, FPNG_DECODE_INVALID_ARG, FPNG_DECODE_FAILED_NOT_PNG,
    FPNG_DECODE_FAILED_HEADER_CRC32, FPNG_DECODE_FAILED_INVALID_DIMENSIONS, FPNG_DECODE_FAILED_DIMENSIONS_TOO_LARGE,
    FPNG_DECODE_FAILED_CHUNK_PARSING, FPNG_DECODE_FAILED_INVALID_IDAT,
    fpng_init, fpng_cpu_supports_sse41, fpng_crc32, fpng_adler32, fpng_encode_image_to_memory,
    fpng_encode_image_to_file, fpng_get_info, fpng_decode_memory, fpng_decode_file,
    train_accumulate_device, create_dynamic_block_prefix, set_static_table,
    max_encoded_size, encode_batch_device, decode_batch_device, decode_batch_host, decode_files, pack_files_for_device, get_info_ex, launch_count,
    FPNGB_DECODE_SHAPE_MISMATCH, get_info_batch_device, decode_packed_device, layout_strides,
    FPNGB_DECODE_OUT_OF_SPACE, decode_packed_ragged_device, ragged_views,
    encode_ragged_device, ragged_slot_offsets, compact_packed_device, encode_png_device, png_slot_offsets,
    encode_labels_device, label_slot_offsets, max_label_encoded_size,
    FPNGB_ENCODE_REDUCE, reduced_slot_offsets, max_reduced_encoded_size,
    FPNGB_DECODE_ADLER_MISMATCH, set_decode_verify, decode_verify,
    normalize_scale_bias, denormalize_scale_bias, typed_layout,
    FPNGB_DECODE_BAD_CROP, FPNGB_RESIZE_ANTIALIAS, decode_packed_resized_device,
    FPNGB_DECODE_UNSUPPORTED_PNG, FPNGB_RESIZE_ANY_PNG, get_png_info,
    FPNGB_PNG_ALL_FORMATS, FPNGB_RESIZE_ALL_PNG_FORMATS, FPNGB_PNG_NATIVE, FPNGB_DTYPE_UINT16, FPNGB_RESIZE_NATIVE,
    FPNGB_PNG_INDEX, FPNGB_DECODE_NOT_INDEXED, FPNGB_RESIZE_NEAREST, FPNGB_RESIZE_NEAREST_EXACT, FPNGB_RESIZE_INDEX,
    FPNGB_RESIZE_BICUBIC,
    FPNGB_VIEW_HFLIP, FPNGB_VIEW_VFLIP, FPNGB_DECODE_BAD_VIEW, decode_packed_views_device, resize_crop_views, letterbox_views,
)
