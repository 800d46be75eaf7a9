"""Python mirror of the reference's operator interface (src/fpng.h:13-111) over the C ABI.

Reference signature                                        -> here
  fpng_init()                                              -> fpng_init(device=-1)
  fpng_encode_image_to_memory(pImage,w,h,chans,out,flags)  -> fpng_encode_image_to_memory(image,w,h,chans,flags) -> (ok, bytes)
  fpng_decode_memory(pImage,size,out,w,h,chans,desired)    -> fpng_decode_memory(data, desired) -> (status, pixels, w, h, chans)
Errors follow the reference: encode returns (False, b"") on invalid arguments, decode returns the FPNG_DECODE_* codes.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import FpngB200Error, LabelPalette, PixelFormat, check, lib

FPNG_ENCODE_SLOWER = 1          # src/fpng.h:38
FPNG_FORCE_UNCOMPRESSED = 2     # src/fpng.h:41
FPNGB_ENCODE_REDUCE = 256       # include/fpng_b200.h: each image in the smallest PNG format that holds it exactly
(FPNG_DECODE_SUCCESS, FPNG_DECODE_NOT_FPNG, FPNG_DECODE_INVALID_ARG, FPNG_DECODE_FAILED_NOT_PNG,
 FPNG_DECODE_FAILED_HEADER_CRC32, FPNG_DECODE_FAILED_INVALID_DIMENSIONS, FPNG_DECODE_FAILED_DIMENSIONS_TOO_LARGE,
 FPNG_DECODE_FAILED_CHUNK_PARSING, FPNG_DECODE_FAILED_INVALID_IDAT, FPNG_DECODE_FILE_OPEN_FAILED,
 FPNG_DECODE_FILE_TOO_LARGE, FPNG_DECODE_FILE_READ_FAILED, FPNG_DECODE_FILE_SEEK_FAILED) = range(13)   # src/fpng.h:57-77


FPNGB_DECODE_ADLER_MISMATCH = 102   # include/fpng_b200.h: verified decode, the zlib Adler-32 does not match the inflated stream


def set_decode_verify(on: bool) -> None:
    """Turns the decoder's integrity check on or off for every later decode call of the process (include/fpng_b200.h,
    fpngb_set_decode_verify): the IDAT CRC-32 (a mismatch gives FPNG_DECODE_FAILED_HEADER_CRC32) and the zlib Adler-32
    (FPNGB_DECODE_ADLER_MISMATCH), both on the GPU.  Off at load: statuses and pixels are then the reference's.  Works before
    fpng_init()."""
    check(lib().fpngb_set_decode_verify(1 if on else 0), "set_decode_verify")


def decode_verify() -> bool:
    """Whether decode calls verify the IDAT CRC-32 and the zlib Adler-32 (set_decode_verify)."""
    return bool(lib().fpngb_get_decode_verify())


def _u8(buf) -> np.ndarray:
    if isinstance(buf, np.ndarray):
        return np.ascontiguousarray(buf).view(np.uint8).reshape(-1)
    return np.frombuffer(bytes(buf), dtype=np.uint8)


def fpng_init(device: int = -1) -> None:
    """src/fpng.h:17. Brings up the CUDA side (device, stream, code books). Raises when no GPU is present."""
    check(lib().fpngb_init(device), "fpng_init")


def fpng_cpu_supports_sse41() -> bool:
    """src/fpng.h:23. Kept for API completeness; this implementation has no CPU SIMD path, so always False."""
    if not lib().fpngb_is_initialized():
        raise FpngB200Error("fpng_cpu_supports_sse41: fpng_init() must be called first")
    return False


def launch_count() -> int:
    return int(lib().fpngb_launch_count())


def max_encoded_size(w: int, h: int, chans: int) -> int:
    return int(lib().fpngb_max_encoded_size(w, h, chans))


def fpng_crc32(data, prev_crc32: int = 0) -> int:
    a = _u8(data)
    return int(lib().fpngb_crc32(a.ctypes.data_as(C.c_void_p), a.size, prev_crc32))


def fpng_adler32(data, adler: int = 1) -> int:
    a = _u8(data)
    return int(lib().fpngb_adler32(a.ctypes.data_as(C.c_void_p), a.size, adler))


def fpng_encode_image_to_memory(image, w: int, h: int, num_chans: int, flags: int = 0):
    """src/fpng.h:48 / src/fpng.cpp:1662.  Returns (ok, png_bytes)."""
    L = lib()
    if w < 1 or h < 1 or num_chans not in (3, 4) or w > (1 << 24) or h > (1 << 24) or w * h > 0xFFFFFFFF:
        return False, b""
    a = _u8(image)
    if a.size != w * h * num_chans:
        return False, b""
    cap = max_encoded_size(w, h, num_chans)
    out = np.empty(cap, dtype=np.uint8)
    n = C.c_size_t(0)
    rc = L.fpngb_encode_host(a.ctypes.data_as(C.c_void_p), w, h, num_chans, flags, out.ctypes.data_as(C.c_void_p), cap, C.byref(n))
    if rc == 1:
        return False, b""
    check(rc, "fpng_encode_image_to_memory")
    return True, out[: n.value].tobytes()


def fpng_encode_image_to_file(filename: str, image, w: int, h: int, num_chans: int, flags: int = 0) -> bool:
    """src/fpng.h:52."""
    ok, data = fpng_encode_image_to_memory(image, w, h, num_chans, flags)
    if not ok:
        return False
    try:
        with open(filename, "wb") as f:
            f.write(data)
    except OSError:
        return False
    return True


def fpng_get_info(data):
    """src/fpng.h:92. Returns (status, w, h, channels_in_file)."""
    a = _u8(data)
    w, h, c = C.c_uint32(), C.c_uint32(), C.c_uint32()
    st = lib().fpngb_get_info(a.ctypes.data_as(C.c_void_p), a.size, C.byref(w), C.byref(h), C.byref(c))
    return st, w.value, h.value, c.value


def fpng_decode_memory(data, desired_channels: int):
    """src/fpng.h:108. Returns (status, pixels|None, w, h, channels_in_file)."""
    a = _u8(data)
    if a.size == 0 or desired_channels not in (3, 4):
        return FPNG_DECODE_INVALID_ARG, None, 0, 0, 0
    st, w, h, c = fpng_get_info(a)
    if st != FPNG_DECODE_SUCCESS:
        return st, None, w, h, c
    need = w * h * desired_channels
    if need > 0xFFFFFFFF:
        return FPNG_DECODE_FAILED_DIMENSIONS_TOO_LARGE, None, w, h, c
    out = np.empty(need, dtype=np.uint8)
    ww, hh, cc = C.c_uint32(), C.c_uint32(), C.c_uint32()
    st = lib().fpngb_decode_host(a.ctypes.data_as(C.c_void_p), a.size, out.ctypes.data_as(C.c_void_p), need,
                                 C.byref(ww), C.byref(hh), C.byref(cc), desired_channels)
    return st, (out if st == 0 else None), ww.value, hh.value, cc.value


def fpng_decode_file(filename: str, desired_channels: int):
    """src/fpng.h:111."""
    try:
        with open(filename, "rb") as f:
            data = f.read()
    except OSError:
        return FPNG_DECODE_FILE_OPEN_FAILED, None, 0, 0, 0
    if len(data) > 0xFFFFFFFF:
        return FPNG_DECODE_FILE_TOO_LARGE, None, 0, 0, 0
    return fpng_decode_memory(data, desired_channels)


def layout_strides(shape, strides, channels=(3, 4)):
    """Byte strides (image_stride, row_pitch, pixel_stride, chan_stride) of an [n, h, w, chans] uint8 view, in the form the
    *_strided C calls take (include/fpng_b200.h, "Pixel layouts").  Two layouts are supported: interleaved (pixel_stride ==
    chans, chan_stride == 1: HWC rows at any pitch) and planar (pixel_stride == 1, chan_stride >= 1: CHW or HCW planes).  The
    stride of a dimension of size 1 is ignored and replaced by the value of a tightly packed batch (w == 1 is interleaved when
    chan_stride == 1, planar otherwise).  Raises ValueError for any other layout.  channels: the channel counts the calling
    entry point takes (1 .. 4 for the native resized decode)."""
    n, h, w, c = (int(v) for v in shape)
    image, row, pixel, chan = (int(v) for v in strides)
    if c not in channels:
        raise ValueError(f"layout_strides: {c} channels ({' or '.join(map(str, channels))} are supported)")
    if min(image, row, pixel, chan) < 0:
        raise ValueError("layout_strides: negative strides are not supported")
    if w == 1:
        pixel = c if chan == 1 else 1
    interleaved = pixel == c and chan == 1
    planar = not interleaved and pixel == 1 and chan >= 1
    if not (interleaved or planar):
        raise ValueError(f"layout_strides: strides {tuple(strides)} of an {tuple(shape)} view are neither interleaved "
                         f"(pixel stride {c}, channel stride 1) nor planar (pixel stride 1, channel stride >= 1)")
    if h == 1:
        row = w * c if interleaved else w
    if n == 1:
        image = h * row
    return image, row, pixel, chan


def _layout(t, shape, channels=(3, 4)):
    """The byte strides (image_stride, row_pitch, pixel_stride, chan_stride) of the C calls for t, an [n, h, w, chans] array of
    the given shape: those of tight rows for a contiguous tensor, else those of a view of that shape in one of the layouts of
    layout_strides.  ValueError for a view of another shape or layout."""
    if t.is_contiguous():
        n, h, w, c = (int(v) for v in shape)
        es = t.element_size()
        return h * w * c * es, w * c * es, c * es, es
    if tuple(t.shape) != tuple(shape):
        raise ValueError(f"a non-contiguous view must have shape {tuple(shape)}, got {tuple(t.shape)}")
    return typed_layout(t.shape, t.stride(), t.element_size(), channels)


def _check_arg(t, name, device, dtype, entries=0, row_bytes=None, view=False):
    """ValueError unless t, the tensor a caller passed as `name`, is a CUDA tensor on `device` of `dtype` that holds what the call
    writes there: with row_bytes (an encode's out), at least `entries` rows of row_bytes with unit stride within a row; with view
    (a decode's pixels), a non-contiguous view, whose shape and layout _layout checks, or else a contiguous tensor of at least
    `entries` elements, as for every other tensor."""
    import torch

    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != device:
        raise ValueError(f"{name}: a CUDA tensor on {device} is needed")
    if t.dtype != dtype:
        raise ValueError(f"{name}: dtype {t.dtype}, {dtype} is needed")
    if row_bytes is not None:
        ok = t.dim() == 2 and t.shape[0] >= entries and t.shape[1] >= row_bytes and (t.stride(1) == 1 or t.shape[1] == 1)
        want = f"at least [{entries}, {row_bytes}] with unit stride within a row"
    else:
        ok = (view and not t.is_contiguous()) or (t.is_contiguous() and t.numel() >= entries)
        want = f"a contiguous tensor of at least {entries} elements" + (" or an [n, h, w, c] view" if view else "")
    if not ok:
        raise ValueError(f"{name}: shape {tuple(t.shape)} with strides {t.stride()}: {want} is needed")


def _stream(stream, device):
    """the stream a call enqueues on: `stream` (a cudaStream_t handle) when given, else the current torch stream of device"""
    import torch

    return stream if stream is not None else torch.cuda.current_stream(device).cuda_stream


def encode_batch_device(images, flags: int = 0, out=None, sizes=None, stream=None, scale=None, bias=None):
    """Encode a batch of equally sized device-resident images.

    images: CUDA tensor [n, h, w, chans]: contiguous, or any view in one of the two layouts of layout_strides -- e.g.
    x_nchw.permute(0, 2, 3, 1), a crop canvas[:, y0:y1, x0:x1, :] or img.expand(n, -1, -1, -1) -- which is read in place,
    without a copy.  torch.uint8 pixels are encoded as they are.  torch.float32 / float16 / bfloat16 elements x of channel c
    are encoded as the bytes nan_to_num(x.float() * scale[c] + bias[c], nan=0).round().clamp(0, 255), rounding half to even,
    converted on the GPU (scale defaults to 1, bias to 0; one value or one per channel; denormalize_scale_bias inverts a
    normalisation): a model's NCHW output in [-1, 1] is encode_batch_device(x.permute(0, 2, 3, 1), scale=127.5, bias=127.5).
    uint8 input takes no scale or bias and other dtypes are refused (ValueError).  Returns (out [n, stride] uint8, sizes [n]
    int32 holding uint32 file sizes) on the same device; kernels are enqueued on the current torch stream (or `stream`), not
    synchronised.
    """
    import torch

    assert images.dim() == 4
    n, h, w, c = images.shape
    fmt = _pixel_format(images.dtype, scale, bias, c, "encode_batch_device")
    assert images.is_cuda
    layout = _layout(images, images.shape)
    cap = max_encoded_size(w, h, c)
    if out is None:
        out = torch.empty((n, (cap + 15) // 16 * 16), dtype=torch.uint8, device=images.device)
    if sizes is None:
        sizes = torch.empty((n,), dtype=torch.int32, device=images.device)
    _check_arg(out, "out", images.device, torch.uint8, n, row_bytes=cap)
    _check_arg(sizes, "sizes", images.device, torch.int32, n)
    args = (images.data_ptr(), *layout, n, w, h, c) + ((C.byref(fmt),) if fmt is not None else ())
    rc = (lib().fpngb_encode_batch_device_strided if fmt is None else lib().fpngb_encode_batch_device_typed)(
        *args, flags, out.data_ptr(), out.stride(0), sizes.data_ptr(), _stream(stream, images.device))
    check(rc, "encode_batch_device")
    return out, sizes


def ragged_slot_offsets(shapes):
    """The slot offsets of encode_ragged_device for images of the given (h, w, chans) shapes: the exclusive prefix of
    max_encoded_size rounded up to 16 bytes, in index order, with the total as the last of the n + 1 entries."""
    return png_slot_offsets([(h, w, c, 8) for (h, w, c) in shapes])


def _encode_images(images, depths, fmt, flags, out, stream, png, what, bound=None):
    """Encodes images, a list of [h, w, c] CUDA tensors of which image i is written at depths[i] bits per sample, with one call
    of fpngb_encode_png_ragged_device (png, dims {w, h, c, depth}) or fpngb_encode_ragged_device (dims {w, h, c}), or of its
    _typed twin when fmt is given.  out defaults to the slot total, a slot being bound(w, h, c, depth) (default: max_encoded_size
    of the pixel bytes) rounded up to 16.  Returns (out, offsets, sizes)."""
    import torch

    # the per-image work here is the host cost of the call: attribute reads only; the layout rules are checked by the C call
    # (an unsupported layout raises FpngB200Error "invalid argument")
    n = len(images)
    ptrs, dims, strides, elem = [], [], [], []
    for t, d in zip(images, depths):
        assert t.is_cuda and t.dim() == 3, "images: [h, w, c] CUDA tensors"
        h, w, c = t.shape
        ptrs.append(t.data_ptr()); dims.append((w, h, c, d)); strides.append(t.stride()); elem.append(t.element_size())
    ptrs = np.array(ptrs, dtype=np.uint64)
    dims = np.array(dims, dtype=np.uint32).reshape(n, 4)
    strides = np.array(strides, dtype=np.uint64).reshape(n, 3) * np.array(elem, dtype=np.uint64).reshape(n, 1)    # in bytes
    device = images[0].device if n else torch.device("cuda")
    if out is None:
        slot = {}
        keys = list(map(tuple, dims.tolist()))
        for key in keys:
            if key not in slot:
                w, h, c, d = key
                slot[key] = ((bound(w, h, c, d) if bound else max_encoded_size(w, h, c * d // 8)) + 15) // 16 * 16
        total = sum(slot[key] for key in keys)
        out = torch.empty((max(total, 16),), dtype=torch.uint8, device=device)[:total]
    _check_arg(out, "out", device, torch.uint8)
    offsets = torch.empty((n + 1,), dtype=torch.int64, device=device)
    sizes = torch.empty((n,), dtype=torch.int32, device=device)
    if not png:                                                          # fpngb_encode_ragged_device's dims are {w, h, c}
        dims = np.ascontiguousarray(dims[:, :3])
    args = (n, ptrs.ctypes.data_as(C.c_void_p), dims.ctypes.data_as(C.c_void_p), strides.ctypes.data_as(C.c_void_p))
    rest = (flags, out.data_ptr(), out.numel(), offsets.data_ptr(), sizes.data_ptr(), _stream(stream, device))
    name = "fpngb_encode_png_ragged_device" if png else "fpngb_encode_ragged_device"
    if fmt is not None:
        rc = getattr(lib(), name + "_typed")(*args, C.byref(fmt), *rest)
    else:
        rc = getattr(lib(), name)(*args, *rest)
    check(rc, what)
    return out, offsets, sizes


def encode_ragged_device(images, flags: int = 0, out=None, stream=None, scale=None, bias=None):
    """Encode device images of ANY shapes, channel counts and layouts in one call (fpngb_encode_ragged_device).

    images: list of CUDA tensors [h, w, chans] (chans 3 or 4), each contiguous or any view in one of the two layouts of
    layout_strides (HWC rows at any pitch, e.g. a crop, or CHW planes, e.g. x_chw.permute(1, 2, 0)); the same tensor may appear
    more than once.  Any other layout raises FpngB200Error (invalid argument).  The images are all torch.uint8, or all one of
    float32 / float16 / bfloat16, converted as in encode_batch_device with scale and bias (one value or one per channel, up to
    the largest channel count of the list); a mixed list raises ValueError.  Returns (out uint8 [total], offsets int64 [n + 1],
    sizes int32 [n]): file i is the sizes[i] bytes at
    out[offsets[i]:], offsets being ragged_slot_offsets of the shapes and offsets[n] the total -- the (data, offsets, sizes)
    decode_packed_ragged_device takes.  out, if given, is a flat 16-byte aligned uint8 CUDA tensor of at least the total; no byte
    of it past the total is written.  Kernels are enqueued on the current torch stream (or `stream`), with no host
    synchronisation."""
    import torch

    n = len(images)
    dtype = images[0].dtype if n else torch.uint8
    mixed = {t.dtype for t in images} - {dtype}
    if mixed:
        raise ValueError(f"encode_ragged_device: the images are all uint8 or all one float dtype, got {dtype} and {mixed.pop()}")
    fmt = _pixel_format(dtype, scale, bias, max((int(t.shape[-1]) for t in images), default=3), "encode_ragged_device")
    return _encode_images(images, [8] * n, fmt, flags, out, stream, False, "encode_ragged_device")


def png_slot_offsets(shapes):
    """The slot offsets of encode_png_device for images of the given (h, w, chans, depth) shapes: the exclusive prefix of
    max_encoded_size(w, h, chans * depth // 8) rounded up to 16 bytes, in index order, with the total as the last of the n + 1
    entries."""
    ofs = np.zeros(len(shapes) + 1, dtype=np.int64)
    for i, (h, w, c, depth) in enumerate(shapes):
        ofs[i + 1] = ofs[i] + (max_encoded_size(int(w), int(h), int(c) * int(depth) // 8) + 15) // 16 * 16
    return ofs


def max_reduced_encoded_size(w: int, h: int, chans: int, depth: int) -> int:
    """fpngb_max_reduced_encoded_size: the slot bound of encode_png_device(reduce=True) for a w x h image of chans channels at
    depth bits: every format the reduction can pick fits, a 256-entry palette with a full tRNS included."""
    if chans not in (1, 2, 3, 4) or depth not in (8, 16):
        raise ValueError(f"max_reduced_encoded_size: chans 1..4 and depth 8 or 16 are needed, got {chans}, {depth}")
    return int(lib().fpngb_max_reduced_encoded_size(w, h, chans, depth))


def reduced_slot_offsets(shapes):
    """The slot offsets of encode_png_device(reduce=True) for images of the given (h, w, chans, depth) shapes: the exclusive
    prefix of max_reduced_encoded_size rounded up to 16 bytes, with the total as the last of the n + 1 entries."""
    ofs = np.zeros(len(shapes) + 1, dtype=np.int64)
    for i, (h, w, c, depth) in enumerate(shapes):
        ofs[i + 1] = ofs[i] + (max_reduced_encoded_size(int(w), int(h), int(c), int(depth)) + 15) // 16 * 16
    return ofs


def _lz77_flags(lz77, name):
    """FPNGB_LZ77_CHAIN(lz77): the flag bits of a chain depth 0 (off) to 256, ValueError otherwise"""
    if isinstance(lz77, bool) or not isinstance(lz77, (int, np.integer)) or not 0 <= int(lz77) <= 256:
        raise ValueError(f"{name}: lz77 is a chain depth from 0 (off) to 256, got {lz77!r}")
    return int(lz77) << 16


def encode_png_device(images, flags: int = 0, out=None, stream=None, scale=None, bias=None, depth=None, reduce=False, lz77=0):
    """Encode device images of 1 to 4 channels to PNG in one call (fpngb_encode_png_ragged_device, or its _typed twin for float
    images).

    images: list of CUDA tensors [h, w, c], c from 1 to 4, each contiguous or a view in one of the layouts of layout_strides (HWC
    rows at any pitch, e.g. a crop, or CHW planes, e.g. x_chw.permute(1, 2, 0)).  Either
      * torch.uint8 (8-bit samples) or torch.uint16 (16-bit samples, written losslessly: depth maps, sensor frames) images, in
        any mix; depth, scale and bias must then be None; or
      * images all of one float dtype, float32, float16 or bfloat16, written at `depth` bits per sample (8 or 16: one value for
        the list or one per image; there is no default, so a depth map is never dropped to 8 bits by accident).  Channel c of
        element x becomes nan_to_num(x.float() * scale[c] + bias[c], nan=0).round().clamp(0, 2**depth - 1), rounding half to
        even, converted on the GPU (scale defaults to 1, bias to 0; one value or one per channel up to the list's largest
        channel count).  Scale and bias are in the output's units: metres to 16-bit millimetres is depth=16, scale=1000.
        Decoding a 16-bit file natively to float32 with scale k and encoding the result with scale 257 / k gives the file back;
        float16 and bfloat16 cannot hold every 16-bit sample.
    The file of an image is byte-identical to the one its quantised uint8 / uint16 image gives: 8-bit images with 3 or 4 channels
    become fpng files, byte-identical to encode_ragged_device's with the same flags; the others (masks, mattes, gray+alpha,
    16-bit) become PNG files with a per-row filter choice and a Huffman code built per image (include/fpng_b200.h).  Other
    dtypes, a mixed float list and the argument combinations above raise ValueError.
    Returns (out uint8 [total], offsets int64 [n + 1], sizes int32 [n]) as encode_ragged_device does, offsets being
    png_slot_offsets of the (h, w, c, depth) shapes -- the (data, offsets, sizes) that decode_packed_ragged_device(any_png=True,
    all_formats=True) reads.  Kernels are enqueued on the current torch stream (or `stream`), with no host synchronisation.

    reduce=True (uint8 / uint16 images only; float images raise ValueError) writes each image in the smallest PNG format that
    holds its pixels exactly, decided on the GPU (include/fpng_b200.h, FPNGB_ENCODE_REDUCE): 1/2/4/8-bit gray, a 1/2/4/8-bit
    palette for at most 256 colours, gray+alpha, RGB or RGBA, at 8 bits when every sample of a uint16 image is a multiple of 257.
    A colour-coded mask becomes a palette file, an RGB binary mask a 1-bit file, an opaque RGBA render an fpng RGB file.  The
    slots are then reduced_slot_offsets of the shapes.  get_info_batch_device / get_png_info report the format written.  The call
    waits once on the host, for the analysis of the images, before it enqueues the encode.

    lz77=K (1 to 256; include/fpng_b200.h, FPNGB_LZ77_CHAIN) writes every image, 8-bit RGB and RGBA included, as a PNG whose
    stream holds LZ77 matches at any distance up to 32 KiB and across rows, found by a hash-chain search of depth K; no fpng
    file is written.  Whether that is smaller than the default files depends on the content (DESIGN §4.6 "LZ77").  Slots and
    offsets are unchanged.  It combines with reduce and FPNG_FORCE_UNCOMPRESSED, not with FPNG_ENCODE_SLOWER.  The files decode
    through the any-PNG inflate, one warp per file."""
    import torch

    flags |= _lz77_flags(lz77, "encode_png_device")
    n = len(images)
    dtypes = {t.dtype for t in images}
    floats = {torch.float32, torch.float16, torch.bfloat16}
    for dt in dtypes:
        if dt not in floats and dt not in (torch.uint8, torch.uint16):
            raise ValueError(f"encode_png_device: torch.uint8, uint16, float32, float16 or bfloat16 images are needed, got {dt}")
    if reduce and dtypes & floats:
        raise ValueError("encode_png_device: reduce=True takes uint8 / uint16 images, not float ones")
    fmt = None
    if dtypes & floats:
        if len(dtypes) > 1:
            raise ValueError(f"encode_png_device: float images are all one dtype, got {sorted(map(str, dtypes))}")
        if depth is None:
            raise ValueError("encode_png_device: float images need depth=8 or depth=16 (one value, or one per image)")
        depths = [depth] * n if np.ndim(depth) == 0 else list(depth)
        if len(depths) != n or any(d not in (8, 16) for d in depths):
            raise ValueError(f"encode_png_device: depth is 8 or 16, one value or one per image ({n}), got {depth}")
        fmt = _pixel_format(images[0].dtype, scale, bias, max(int(t.shape[-1]) for t in images), "encode_png_device")
    elif depth is not None or scale is not None or bias is not None:
        raise ValueError("encode_png_device: depth, scale and bias apply to float images only; uint8 / uint16 are taken as they are")
    depths = depths if fmt is not None else [8 * t.element_size() for t in images]
    if reduce:
        return _encode_images(images, depths, None, flags | FPNGB_ENCODE_REDUCE, out, stream, True, "encode_png_device",
                              bound=lambda w, h, c, d: max_reduced_encoded_size(w, h, c, d))
    return _encode_images(images, depths, fmt, flags, out, stream, True, "encode_png_device")


def _label_palettes(palette, n):
    """The per-image palettes of encode_labels_device as uint8 [K, 3 | 4] numpy arrays (None: gray), ValueError otherwise."""
    if palette is None:
        return [None] * n
    if isinstance(palette, (list, tuple)):
        if len(palette) != n:
            raise ValueError(f"encode_labels_device: palette is one array or a list of {n} (one per image), got {len(palette)}")
        pals = list(palette)
    else:
        pals = [palette] * n
    out = []
    for p in pals:
        if p is None:
            out.append(None)
            continue
        if hasattr(p, "detach"):
            p = p.detach().cpu().numpy()
        a = np.asarray(p)
        if a.dtype != np.uint8 or a.ndim != 2 or a.shape[1] not in (3, 4) or not 1 <= a.shape[0] <= 256:
            raise ValueError(f"encode_labels_device: a palette is a uint8 array of shape [K, 3 or 4] with 1 <= K <= 256, got "
                             f"{a.dtype} {a.shape}")
        out.append(np.ascontiguousarray(a))
    return out


def _palette_struct(a):
    return LabelPalette(None, 0, 0) if a is None else LabelPalette(a.ctypes.data, a.shape[0], a.shape[1])


def _pil_depth(k):
    """PIL's bit depth for a palette of k entries"""
    return 1 if k <= 2 else 2 if k <= 4 else 4 if k <= 16 else 8


def max_label_encoded_size(w: int, h: int, depth: int, palette=None) -> int:
    """fpngb_max_label_encoded_size: the slot bound of a w x h label map at `depth` bits with an optional [K, 3 | 4] palette"""
    pal = _label_palettes(palette, 1)[0]
    return lib().fpngb_max_label_encoded_size(w, h, depth, C.byref(_palette_struct(pal)))


def label_slot_offsets(shapes, palettes=None):
    """The slot offsets of encode_labels_device for label maps of the given (h, w, depth) shapes, with palettes None (all gray)
    or one [K, 3 | 4] array (or None) per map: the exclusive prefix of max_label_encoded_size rounded up to 16 bytes, with the
    total as the last of the n + 1 entries."""
    pals = palettes if palettes is not None else [None] * len(shapes)
    ofs = np.zeros(len(shapes) + 1, dtype=np.int64)
    for i, ((h, w, depth), pal) in enumerate(zip(shapes, pals)):
        ofs[i + 1] = ofs[i] + (max_label_encoded_size(int(w), int(h), int(depth), pal) + 15) // 16 * 16
    return ofs


def encode_labels_device(images, palette=None, depth=None, flags: int = 0, out=None, stream=None, lz77=0):
    """Encode label maps (class ids, masks) on the GPU to palette or gray PNGs in one call (fpngb_encode_label_ragged_device).

    images: list of CUDA tensors [h, w] or [h, w, 1], torch.uint8 or torch.int64 ids (the output of logits.argmax(1)[i] goes in
    as it is), contiguous or a view whose ids are contiguous within a row, at any row pitch (a crop, an expand of one row).
    palette: None (gray files), one uint8 array [K, 3 | 4] (RGB or RGBA, K <= 256) for every image, or a list with one such
    array or None per image.  depth: bits per id, one
    value or one per image; for a palette image it defaults to PIL's rule (K <= 2: 1, <= 4: 2, <= 16: 4, else 8); a gray image
    needs it (1, 2, 4, 8 or 16, 16 only from int64), so that a mask is never truncated by accident.  flags: 0 or
    FPNG_FORCE_UNCOMPRESSED.  An image holding an id outside [0, 2^depth) (gray) or [0, K) (palette) gets size 0; the others are
    unaffected.  Returns (out uint8 [total], offsets int64 [n + 1], sizes int32 [n]) as encode_png_device does, offsets being
    label_slot_offsets -- the (data, offsets, sizes) decode_packed_ragged_device(any_png=True, all_formats=True) reads, with
    indices=True giving the ids back.  Kernels are enqueued on the current torch stream (or `stream`), with no host
    synchronisation.  Other dtypes, shapes and argument values raise ValueError.  lz77=K (1 to 256): the LZ77 mode of
    encode_png_device."""
    import torch

    lz_flags = _lz77_flags(lz77, "encode_labels_device")
    n = len(images)
    if n == 0:
        raise ValueError("encode_labels_device: at least one image is needed")
    pals = _label_palettes(palette, n)
    depths = [depth] * n if depth is None or np.ndim(depth) == 0 else list(depth)
    if len(depths) != n:
        raise ValueError(f"encode_labels_device: depth is one value or one per image ({n}), got {depth}")
    ptrs, dims, strides = [], [], []
    for i, t in enumerate(images):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise ValueError("encode_labels_device: images are CUDA tensors")
        if t.dtype not in (torch.uint8, torch.int64):
            raise ValueError(f"encode_labels_device: torch.uint8 or torch.int64 ids are needed, got {t.dtype}")
        if not (t.dim() == 2 or (t.dim() == 3 and t.shape[2] == 1)):
            raise ValueError(f"encode_labels_device: images are [h, w] or [h, w, 1], got {tuple(t.shape)}")
        h, w = int(t.shape[0]), int(t.shape[1])
        d, pal = depths[i], pals[i]
        if d is None:
            if pal is None:
                raise ValueError("encode_labels_device: gray label maps need depth (1, 2, 4, 8 or 16)")
            d = _pil_depth(pal.shape[0])
        d = int(d)
        if pal is None and d not in (1, 2, 4, 8, 16):
            raise ValueError(f"encode_labels_device: gray depth is 1, 2, 4, 8 or 16, got {d}")
        if pal is not None and (d not in (1, 2, 4, 8) or pal.shape[0] > 1 << d):
            raise ValueError(f"encode_labels_device: a palette of {pal.shape[0]} entries needs depth 1, 2, 4 or 8 with K <= 2^depth, "
                             f"got {d}")
        if t.dtype == torch.uint8 and d > 8:
            raise ValueError("encode_labels_device: depth 16 needs int64 ids")
        es = t.element_size()
        ptrs.append(t.data_ptr()); dims.append((w, h, d, es)); strides.append((t.stride(0) * es, t.stride(1) * es))
        depths[i] = d
    device = images[0].device
    if any(t.device != device for t in images):
        raise ValueError("encode_labels_device: the images are on one device")
    if flags & ~FPNG_FORCE_UNCOMPRESSED:
        raise ValueError("encode_labels_device: flags is 0 or FPNG_FORCE_UNCOMPRESSED")
    if min(s for st in strides for s in st) < 0:
        raise ValueError("encode_labels_device: negative strides are not supported")
    structs = (LabelPalette * n)(*[_palette_struct(p) for p in pals])
    if out is None:
        total = int(label_slot_offsets([(dm[1], dm[0], dm[2]) for dm in dims], pals)[-1])
        out = torch.empty((max(total, 16),), dtype=torch.uint8, device=device)[:total]
    _check_arg(out, "out", device, torch.uint8)
    offsets = torch.empty((n + 1,), dtype=torch.int64, device=device)
    sizes = torch.empty((n,), dtype=torch.int32, device=device)
    ptrs = np.array(ptrs, dtype=np.uint64)
    dims = np.array(dims, dtype=np.uint32).reshape(n, 4)
    strides = np.array(strides, dtype=np.uint64).reshape(n, 2)
    rc = lib().fpngb_encode_label_ragged_device(n, ptrs.ctypes.data_as(C.c_void_p), dims.ctypes.data_as(C.c_void_p),
                                                strides.ctypes.data_as(C.c_void_p), C.cast(structs, C.c_void_p), flags | lz_flags,
                                                out.data_ptr(), out.numel(), offsets.data_ptr(), sizes.data_ptr(),
                                                _stream(stream, device))
    check(rc, "encode_labels_device")
    return out, offsets, sizes


def compact_packed_device(data, offsets, sizes, out=None, stream=None):
    """Pack the files of a packed device buffer (file i: sizes[i] bytes at data[offsets[i]:], every offset a multiple of 16, e.g.
    an encode_ragged_device result) back to back, each starting 16-byte aligned (fpngb_compact_packed_device).  Returns
    (out uint8, dst_offsets int64 [n + 1]): file i at out[dst_offsets[i]:], dst_offsets[n] the total, with bit 63 set (a negative
    value) when out was too small -- the files that did not fit are not copied.  out defaults to data.numel() bytes, which holds
    every compaction of files that do not overlap.  Stream-ordered, no host synchronisation."""
    import torch

    n = _packed_args(data, offsets, sizes)
    if out is None:
        out = torch.empty((max(data.numel(), 16),), dtype=torch.uint8, device=data.device)
    _check_arg(out, "out", data.device, torch.uint8)
    dst_offsets = torch.empty((n + 1,), dtype=torch.int64, device=data.device)
    s = _stream(stream, data.device)
    check(lib().fpngb_compact_packed_device(data.data_ptr(), offsets.data_ptr(), sizes.data_ptr(), n, out.data_ptr(), out.numel(),
                                            dst_offsets.data_ptr(), s), "compact_packed_device")
    return out, dst_offsets


_DTYPE_CODES = {"float32": 1, "float16": 2, "bfloat16": 3}   # FPNGB_DTYPE_*


def _out_dtype(out, dtype):
    """the output dtype of a decode call: out's when given (dtype must then agree), else dtype, else torch.uint8"""
    import torch

    if out is not None:
        if dtype is not None and dtype != out.dtype:
            raise ValueError(f"dtype {dtype} differs from out.dtype {out.dtype}")
        return out.dtype
    return torch.uint8 if dtype is None else dtype


def _per_channel(v, desired_channels, default, what):
    if v is None:
        return [default] * desired_channels
    a = np.asarray(v.detach().cpu().numpy() if hasattr(v, "detach") else v, dtype=np.float32).reshape(-1)
    if a.size == 1:
        a = np.repeat(a, desired_channels)
    if a.size != desired_channels:
        raise ValueError(f"{what}: one value or one per output channel ({desired_channels}), got {a.size}")
    return [float(x) for x in a]


def _pixel_format(dtype, scale, bias, chans, what="pixel format"):
    """None for uint8 pixels (the uint8 calls, which take no scale or bias), else the fpngb_pixel_format of float32 / float16 /
    bfloat16 pixels of chans channels: scale defaults to 1 and bias to 0 per channel; a single value applies to every channel.
    Values are rounded to float32.  ValueError for any other dtype."""
    import torch

    if dtype == torch.uint8:
        if scale is not None or bias is not None:
            raise ValueError(f"{what}: scale and bias apply to float32 / float16 / bfloat16 pixels only; uint8 pixels are taken as they are")
        return None
    code = _DTYPE_CODES.get(str(dtype).replace("torch.", ""))
    if code is None:
        raise ValueError(f"{what}: dtype {dtype}: torch.uint8, float32, float16 or bfloat16")
    fmt = PixelFormat()
    fmt.dtype = code
    fmt.scale[:chans] = _per_channel(scale, chans, 1.0, "scale")
    fmt.bias[:chans] = _per_channel(bias, chans, 0.0, "bias")
    return fmt


def typed_layout(shape, strides, element_size, channels=(3, 4)):
    """Byte strides (image_stride, row_pitch, pixel_stride, chan_stride) of an [n, h, w, chans] view whose elements are
    element_size bytes, as the *_typed C calls take them: layout_strides applied to the element strides torch reports, then
    multiplied by the element size.  NCHW float output is torch.empty(n, c, h, w, dtype=...).permute(0, 2, 3, 1)."""
    return tuple(v * int(element_size) for v in layout_strides(shape, strides, channels))


def normalize_scale_bias(mean, std, max_value=255.0):
    """The (scale, bias) pair, float32 arrays, for which the typed decode computes (x - mean) / std of x = v / max_value:
    scale = 1 / (max_value * std) and bias = -mean / std, computed in float64 and then rounded to float32.  ImageNet:
    normalize_scale_bias((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)).

    The decode computes v * scale + bias (two rounded fp32 operations), not torchvision's Normalize(mean, std)(v / 255), which
    divides, subtracts and divides again; the results can therefore differ in the last bits."""
    m = np.asarray(mean, dtype=np.float64).reshape(-1)
    sd = np.asarray(std, dtype=np.float64).reshape(-1)
    return (1.0 / (float(max_value) * sd)).astype(np.float32), (-m / sd).astype(np.float32)


def denormalize_scale_bias(mean, std, max_value=255.0):
    """The (scale, bias) pair, float32 arrays, that the typed encode applies to a normalised tensor x = (v / max_value - mean) / std
    to get back v: scale = max_value * std and bias = max_value * mean, computed in float64 and then rounded to float32 -- the
    inverse of normalize_scale_bias.  The encode rounds x * scale + bias half to even and clamps it to [0, 255], so a decode with
    normalize_scale_bias(mean, std) followed by an encode with these values gives back the bytes wherever the float type keeps
    enough precision (bfloat16 with CLIP's mean and std misses one value in 768)."""
    m = np.asarray(mean, dtype=np.float64).reshape(-1)
    sd = np.asarray(std, dtype=np.float64).reshape(-1)
    return (float(max_value) * sd).astype(np.float32), (float(max_value) * m).astype(np.float32)


def get_info_ex(data):
    """fpng_get_info plus (idat_ofs, idat_len): the host-side container walk (src/fpng.cpp:2930-3077)."""
    a = _u8(data)
    w, h, c, o, l = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
    st = lib().fpngb_get_info_ex(a.ctypes.data_as(C.c_void_p), a.size, C.byref(w), C.byref(h), C.byref(c), C.byref(o), C.byref(l))
    return st, w.value, h.value, c.value, o.value, l.value


FPNGB_DECODE_UNSUPPORTED_PNG = 104   # any_png decodes: a well-formed PNG the GPU decoder does not read (palette, 16-bit, Adam7, tRNS)
FPNGB_PNG_ALL_FORMATS = 1            # all_formats=True: palette, 1/2/4/16-bit, color-keyed and Adam7 files decode too
FPNGB_PNG_NATIVE = 4                 # native=True: each file at its own channel count, uint16 output, 1 / 2 channels
FPNGB_DTYPE_UINT16 = 4               # fpngb_pixel_format.dtype of uint16 output (native calls only)
FPNGB_PNG_INDEX = 8                  # indices=True: each pixel's raw sample (palette index, gray sample), uint8 or uint16
FPNGB_DECODE_NOT_INDEXED = 105       # indices=True: the file has no single sample the output type holds (fpng, color, 16-bit to uint8)


def get_png_info(data, all_formats=False):
    """get_info_ex with the general-PNG rules of the any_png decodes: fpng files give get_info_ex's row, files the fpng walk
    rejects with FPNG_DECODE_NOT_FPNG are walked again as general PNGs (include/fpng_b200.h): status 0 with the file's own
    channel count (1 gray, 2 gray+alpha, 3, 4), the offset of the first IDAT chunk and the sum of the IDAT data lengths, or
    FPNGB_DECODE_UNSUPPORTED_PNG / a walk error.  all_formats=True applies the walk rules of FPNGB_PNG_ALL_FORMATS: palette,
    1/2/4/16-bit, tRNS and Adam7 files pass too (chans: palette 3, a tRNS chunk in gray / RGB / palette files adds alpha)."""
    a = _u8(data)
    w, h, c, o, l = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
    st = lib().fpngb_get_png_info_ex(a.ctypes.data_as(C.c_void_p), a.size, FPNGB_PNG_ALL_FORMATS if all_formats else 0, C.byref(w),
                                     C.byref(h), C.byref(c), C.byref(o), C.byref(l))
    return st, w.value, h.value, c.value, o.value, l.value


def _all_formats_check(any_png, all_formats, fn, native=False):
    if all_formats and not any_png:
        raise ValueError(f"{fn}: all_formats=True needs any_png=True")
    if native and not any_png:
        raise ValueError(f"{fn}: native=True needs any_png=True")


def _indices_check(indices, any_png, all_formats, native, desired_channels, dtype, fn):
    """ValueError unless an indices=True call is any_png, all_formats and native, at 1 channel, into uint8 or uint16"""
    import torch

    if not indices:
        return
    if not (any_png and all_formats and native):
        raise ValueError(f"{fn}: indices=True needs any_png=True, all_formats=True and native=True")
    if desired_channels != 1:
        raise ValueError(f"{fn}: indices=True needs desired_channels=1, got {desired_channels}")
    if dtype not in (torch.uint8, torch.uint16):
        raise ValueError(f"{fn}: indices=True stores ids as torch.uint8 or torch.uint16, not {dtype}")


def _native_format(dtype, scale, bias, desired_channels, what):
    """the fmt of a native call: None for uint8, FPNGB_DTYPE_UINT16 for uint16 (no scale or bias: ValueError), else _pixel_format's
    over the channels the call may write (4 for desired_channels 0)"""
    import torch

    if dtype == torch.uint16:
        if scale is not None or bias is not None:
            raise ValueError(f"{what}: scale and bias apply to float32 / float16 / bfloat16 pixels only; uint16 pixels are taken as they are")
        fmt = PixelFormat()
        fmt.dtype = FPNGB_DTYPE_UINT16
        return fmt
    return _pixel_format(dtype, scale, bias, desired_channels or 4, what)


def pack_files_for_device(files, device=None):
    """Container-walks a list of fpng files (bytes) of identical dimensions on the host and packs them into one device
    tensor [n, stride].  Returns (tensor, stride, sizes, idat_ofs, idat_len, w, h, chans)."""
    import torch

    infos = [get_info_ex(f) for f in files]
    for st, *_ in infos:
        if st != 0:
            raise FpngB200Error(f"pack_files_for_device: fpng_get_info returned {st}")
    w, h, c = infos[0][1:4]
    if any(i[1:4] != (w, h, c) for i in infos):
        raise FpngB200Error("pack_files_for_device: files differ in dimensions/channels")
    stride = (max(len(f) for f in files) + 16 + 15) // 16 * 16
    host = np.zeros((len(files), stride), dtype=np.uint8)
    for i, f in enumerate(files):
        host[i, : len(f)] = np.frombuffer(f, dtype=np.uint8)
    t = torch.from_numpy(host)
    if device is not None:
        t = t.to(device)
    sizes = np.array([len(f) for f in files], dtype=np.uint32)
    ofs = np.array([i[4] for i in infos], dtype=np.uint32)
    lens = np.array([i[5] for i in infos], dtype=np.uint32)
    return t, stride, sizes, ofs, lens, w, h, c


def decode_batch_device(files_dev, sizes, idat_ofs, idat_len, w: int, h: int, chans_in_file: int, desired_channels: int,
                        out=None, status=None, stream=None, dtype=None, scale=None, bias=None):
    """Decode n fpng files resident on the device (tensor [n, stride] uint8). Returns (pixels [n, h, w, desired], status [n]).
    out may be any non-overlapping [n, h, w, desired] view in one of the two layouts of layout_strides, e.g.
    torch.empty(n, desired, h, w).permute(0, 2, 3, 1) for NCHW pixels; the kernels write it in place.
    The output dtype is out.dtype when out is given, else dtype (default torch.uint8).  torch.float32 / float16 / bfloat16 store
    T(v * scale[c] + bias[c]) for every uint8 value v of channel c, converted in the decoder's last kernel (scale defaults to 1,
    bias to 0; one value or one per channel; normalize_scale_bias turns a mean / std into them).  uint8 output takes no scale
    or bias (ValueError)."""
    import torch

    assert files_dev.is_cuda and files_dev.dtype == torch.uint8 and files_dev.dim() == 2 and files_dev.is_contiguous()
    n, dev = files_dev.shape[0], files_dev.device
    odt = _out_dtype(out, dtype)
    fmt = _pixel_format(odt, scale, bias, desired_channels, "decode_batch_device")
    shape = (n, h, w, desired_channels)
    if out is None:
        out = torch.empty(shape, dtype=odt, device=dev)
    if status is None:
        status = torch.empty((n,), dtype=torch.int32, device=dev)
    _check_arg(out, "out", dev, odt, n * h * w * desired_channels, view=True)
    _check_arg(status, "status", dev, torch.int32, n)
    sizes = np.ascontiguousarray(sizes, dtype=np.uint32); idat_ofs = np.ascontiguousarray(idat_ofs, dtype=np.uint32)
    idat_len = np.ascontiguousarray(idat_len, dtype=np.uint32)
    args = (files_dev.data_ptr(), files_dev.stride(0), sizes.ctypes.data_as(C.c_void_p), idat_ofs.ctypes.data_as(C.c_void_p),
            idat_len.ctypes.data_as(C.c_void_p), n, w, h, chans_in_file, desired_channels, out.data_ptr(), *_layout(out, shape))
    args += (C.byref(fmt),) if fmt is not None else ()
    rc = (lib().fpngb_decode_batch_device_strided if fmt is None else lib().fpngb_decode_batch_device_typed)(
        *args, status.data_ptr(), _stream(stream, dev))
    check(rc, "decode_batch_device")
    return out, status


FPNGB_DECODE_SHAPE_MISMATCH = 100   # decode_packed_device only: a valid file whose w/h/chans differ from the call's


def _packed_args(data, offsets, sizes):
    import torch

    assert data.is_cuda and data.dtype == torch.uint8 and data.is_contiguous(), "data: flat uint8 CUDA tensor"
    assert offsets.is_cuda and offsets.dtype == torch.int64 and offsets.is_contiguous(), "offsets: int64 CUDA tensor"
    assert sizes.is_cuda and sizes.dtype == torch.int32 and sizes.is_contiguous() and sizes.dim() == 1, "sizes: int32 CUDA tensor"
    n = sizes.shape[0]
    assert offsets.numel() >= n, "one offset per file (dist.compact's extra total at the end is ignored)"
    return n


def get_info_batch_device(data, offsets, sizes, stream=None, any_png=False, all_formats=False):
    """Container walk on the device of the files packed in `data` (file i: sizes[i] bytes at offsets[i]) -- the layout of
    dist.compact and of the gather window.  data: flat uint8 CUDA tensor, offsets: int64 CUDA tensor (>= n entries),
    sizes: int32 CUDA tensor [n] (uint32 values; 0 = no file).  Returns an int32 CUDA tensor [n, 6]: per file
    (status, w, h, chans, idat_ofs, idat_len) as get_info_ex (any_png: as get_png_info, with all_formats as get_png_info's).
    Enqueued on the current torch stream (or `stream`); no host synchronisation."""
    import torch

    _all_formats_check(any_png, all_formats, "get_info_batch_device")
    n = _packed_args(data, offsets, sizes)
    info = torch.empty((n, 6), dtype=torch.int32, device=data.device)
    if n == 0:
        return info
    s = _stream(stream, data.device)
    if all_formats:
        rc = lib().fpngb_get_png_info_batch_device_ex(data.data_ptr(), offsets.data_ptr(), sizes.data_ptr(), n, FPNGB_PNG_ALL_FORMATS,
                                                      info.data_ptr(), s)
    else:
        fn = lib().fpngb_get_png_info_batch_device if any_png else lib().fpngb_get_info_batch_device
        rc = fn(data.data_ptr(), offsets.data_ptr(), sizes.data_ptr(), n, info.data_ptr(), s)
    check(rc, "get_info_batch_device")
    return info


def decode_packed_device(data, offsets, sizes, w: int, h: int, chans_in_file: int, desired_channels: int, max_file_size=None,
                         out=None, status=None, stream=None, dtype=None, scale=None, bias=None):
    """Decode the w x h x chans_in_file fpng files packed in device memory (same arguments as get_info_batch_device; every
    file 4-byte aligned).  The container walk runs on the device: no host synchronisation and no host copy.
    Returns (pixels uint8 [n, h, w, desired_channels], status int32 [n]); out may be a strided view as in decode_batch_device.  status[i] is fpng_decode_memory's code for file i,
    or FPNGB_DECODE_SHAPE_MISMATCH for a valid file of another shape, or FPNG_DECODE_INVALID_ARG for size 0, size >
    max_file_size or an offset that is not a multiple of 4; pixels of files with a non-zero status are left untouched.
    max_file_size (bytes) bounds every file and sizes the decoder's workspace; the default, max_encoded_size(w, h,
    chans_in_file), holds for every file this library or the reference encoder writes.  A smaller bound known to the
    caller saves workspace and launch overhead.  dtype, scale and bias as in decode_batch_device."""
    import torch

    n = _packed_args(data, offsets, sizes)
    if max_file_size is None:
        max_file_size = min(max_encoded_size(w, h, chans_in_file), 0xFFFFFFFF)
    odt = _out_dtype(out, dtype)
    fmt = _pixel_format(odt, scale, bias, desired_channels, "decode_packed_device")
    shape = (n, h, w, desired_channels)
    if out is None:
        out = torch.empty(shape, dtype=odt, device=data.device)
    if status is None:
        status = torch.empty((n,), dtype=torch.int32, device=data.device)
    _check_arg(out, "out", data.device, odt, n * h * w * desired_channels, view=True)
    _check_arg(status, "status", data.device, torch.int32, n)
    args = (data.data_ptr(), offsets.data_ptr(), sizes.data_ptr(), n, max_file_size, w, h, chans_in_file, desired_channels,
            out.data_ptr(), *_layout(out, shape))
    args += (C.byref(fmt),) if fmt is not None else ()
    rc = (lib().fpngb_decode_packed_device_strided if fmt is None else lib().fpngb_decode_packed_device_typed)(
        *args, status.data_ptr(), _stream(stream, data.device))
    check(rc, "decode_packed_device")
    return out, status


FPNGB_DECODE_OUT_OF_SPACE = 101    # decode_packed_ragged_device only: the file's pixels do not fit in `out`


def _ragged_bounds(data, offsets, sizes, n, desired_channels, max_file_size, max_w, max_h, stream, element_size=1, any_png=False,
                   all_formats=False):
    """The bounds of decode_packed_ragged_device the caller left out, and the exact output size in bytes they give for elements
    of element_size bytes: one device walk (get_info_batch_device) and one read-back of (info, sizes, offsets), which
    synchronises with the stream.  desired_channels 0 (native calls) sizes each file at its info row's channel count."""
    import torch

    info = get_info_batch_device(data, offsets, sizes, stream, any_png=any_png, all_formats=all_formats)
    if stream is not None:
        torch.cuda.ExternalStream(stream, device=data.device).synchronize()
    t = torch.cat([info.long(), (sizes.long() & 0xFFFFFFFF)[:, None], offsets[:n, None]], 1).cpu().numpy()
    st, w, h, size, ofs = t[:, 0], t[:, 1], t[:, 2], t[:, 6], t[:, 7]
    walked = st == 0
    if max_file_size is None:
        max_file_size = int(size[walked].max()) if walked.any() else 1
    if max_w is None:
        max_w = int(w[walked].max()) if walked.any() else 1
    if max_h is None:
        max_h = int(h[walked].max()) if walked.any() else 1
    px = w * h * (desired_channels if desired_channels else t[:, 3])
    placed = (walked & (size <= max_file_size) & (ofs % 4 == 0) & (ofs + size <= data.numel()) & (w <= max_w) & (h <= max_h)
              & (px <= 0xFFFFFFFF))
    total = int(((px[placed] * element_size + 15) // 16 * 16).sum())
    return max_file_size, max_w, max_h, total


def decode_packed_ragged_device(data, offsets, sizes, desired_channels: int, out=None, max_file_size=None, max_w=None, max_h=None,
                                stream=None, dtype=None, scale=None, bias=None, any_png=False, all_formats=False, native=False,
                                indices=False):
    """Decode fpng files of ANY shapes and channel counts packed in device memory (the layout of get_info_batch_device; base_bytes
    is data.numel()) in one call, pixels placed back to back.  Returns (out uint8 [out_cap], out_offsets int64 [n + 1],
    info int32 [n, 6], status int32 [n]):
      * file i's pixels are the h*w*desired_channels bytes at out[out_offsets[i]:], tight HWC rows (ragged_views cuts them out);
        every decodable file takes its size rounded up to 16 bytes, in index order; out_offsets[n] is the total, with bit 63 set
        (a negative value) when it exceeds out.numel(), and a file that does not fit gets FPNGB_DECODE_OUT_OF_SPACE;
      * info[i] is get_info_batch_device's row for file i ({FPNG_DECODE_INVALID_ARG, 0, ...} when its arguments fail);
      * status[i] is fpng_decode_memory's code, FPNG_DECODE_INVALID_ARG for size 0, size > max_file_size, offset % 4 != 0 or a
        file that runs past the end of data, FPNGB_DECODE_SHAPE_MISMATCH for a valid file wider than max_w or taller than
        max_h, or FPNGB_DECODE_OUT_OF_SPACE.  Bytes of out outside the decoded files are left untouched.
    With `out` (a flat, 16-byte aligned uint8 CUDA tensor) and all three bounds given, the call is stream-ordered: no host
    synchronisation.  Any of them that is None is computed from one get_info_batch_device and one read-back to the host, which
    waits for the stream: max_file_size, max_w and max_h become the largest size, width and height of the files the container
    walk accepts, and out is allocated at the exact total.  Tight bounds save workspace and launch overhead.
    dtype, scale and bias as in decode_batch_device: with a float output, out is a flat tensor of that dtype, file i takes
    align_up(h*w*desired_channels*element_size, 16) bytes, and out_offsets stay in bytes (ragged_views converts them).
    any_png=True also decodes, on the GPU, the 8-bit non-interlaced gray, gray+alpha, RGB and RGBA PNGs of any other writer
    (fpngb_decode_packed_png_device): their info rows are get_png_info's, their statuses 0, FPNGB_DECODE_UNSUPPORTED_PNG, a walk
    error or FPNG_DECODE_FAILED_INVALID_IDAT for a bad stream; fpng files decode exactly as without it.
    all_formats=True (with any_png=True, else ValueError) also decodes palette, 1/2/4-bit gray, 16-bit, color-keyed (tRNS) and
    Adam7-interlaced files (FPNGB_PNG_ALL_FORMATS; pixel rules in include/fpng_b200.h): sub-byte gray scaled to 0..255, 16-bit
    samples as their high byte (typed output: s / 257), palette entries with tRNS alpha, a color key as alpha 0.
    native=True (with any_png=True, else ValueError) decodes each file at its own channel count and bit depth (FPNGB_PNG_NATIVE;
    rules in include/fpng_b200.h): desired_channels may also be 1 (gray, or the luma of color files: Pillow's convert("L")), 2
    (with alpha) or 0 / None (each file's own channels, info[i, 3]; ragged_views(..., 0) cuts them), and dtype torch.uint16
    stores 16-bit samples as they are and 8-bit values v as v * 257 (no scale or bias).  Without native those values raise
    ValueError.
    indices=True (FPNGB_PNG_INDEX; needs any_png, all_formats and native, desired_channels=1 and dtype uint8 or uint16, else
    ValueError) decodes label maps: each pixel's raw sample, with no scaling, palette lookup or alpha.  Palette files give their
    indices (np.asarray(PIL.Image.open(f)) for PIL mode "P"), gray files of any depth their samples (a 1-bit mask 0 / 1, a 4-bit
    one 0..15).  fpng files, color files and 16-bit gray into uint8 get FPNGB_DECODE_NOT_INDEXED, take no space and are not
    decoded."""
    import torch

    _all_formats_check(any_png, all_formats, "decode_packed_ragged_device", native)
    odt = _out_dtype(out, dtype)
    _indices_check(indices, any_png, all_formats, native, desired_channels, odt, "decode_packed_ragged_device")
    if native:
        desired_channels = desired_channels or 0
        if desired_channels not in (0, 1, 2, 3, 4):
            raise ValueError(f"decode_packed_ragged_device: desired_channels {desired_channels}: 0 (None), 1, 2, 3 or 4")
        fmt = _native_format(odt, scale, bias, desired_channels, "decode_packed_ragged_device")
    else:
        if desired_channels in (0, 1, 2, None):
            raise ValueError(f"decode_packed_ragged_device: desired_channels {desired_channels} needs native=True")
        assert desired_channels in (3, 4), "desired_channels: 3 or 4"
        fmt = _pixel_format(odt, scale, bias, desired_channels, "decode_packed_ragged_device")
    n = _packed_args(data, offsets, sizes)
    es = torch.empty((), dtype=odt).element_size()
    if out is None or max_file_size is None or max_w is None or max_h is None:
        max_file_size, max_w, max_h, total = _ragged_bounds(data, offsets, sizes, n, desired_channels, max_file_size, max_w, max_h,
                                                             stream, es, any_png, all_formats)
        if out is None:
            out = torch.empty((max(total, 16) // es,), dtype=odt, device=data.device)[:total // es]
    _check_arg(out, "out", data.device, odt)
    out_offsets = torch.empty((n + 1,), dtype=torch.int64, device=data.device)
    info = torch.empty((n, 6), dtype=torch.int32, device=data.device)
    status = torch.empty((n,), dtype=torch.int32, device=data.device)
    s = _stream(stream, data.device)
    args = (data.data_ptr(), data.numel(), offsets.data_ptr(), sizes.data_ptr(), n, min(int(max_file_size), 0xFFFFFFFF), int(max_w),
            int(max_h), desired_channels, out.data_ptr(), out.numel() * es, out_offsets.data_ptr(), info.data_ptr())
    if all_formats or native:
        rc = lib().fpngb_decode_packed_png_device_ex(*args, (FPNGB_PNG_ALL_FORMATS if all_formats else 0) |
                                                     (FPNGB_PNG_NATIVE if native else 0) | (FPNGB_PNG_INDEX if indices else 0),
                                                     None if fmt is None else C.byref(fmt),
                                                     status.data_ptr(), s)
    elif any_png:
        rc = lib().fpngb_decode_packed_png_device(*args, None if fmt is None else C.byref(fmt), status.data_ptr(), s)
    elif fmt is None:
        rc = lib().fpngb_decode_packed_ragged_device(*args, status.data_ptr(), s)
    else:
        rc = lib().fpngb_decode_packed_ragged_device_typed(*args, C.byref(fmt), status.data_ptr(), s)
    check(rc, "decode_packed_ragged_device")
    return out, out_offsets, info, status


def ragged_views(out, out_offsets, info, status, desired_channels: int):
    """Per file of a decode_packed_ragged_device result, an [h, w, desired_channels] view into `out` (any dtype: the byte offsets
    become element offsets), or None when the file's status is not 0.  desired_channels 0 (or None: a native call's) takes each
    file's info row channel count.  Reads out_offsets, info and status back to the host, so it waits for the device."""
    offs = out_offsets.cpu().numpy()
    inf = info.cpu().numpy()
    st = status.cpu().numpy()
    views = []
    for i in range(st.shape[0]):
        if st[i] != 0:
            views.append(None)
            continue
        w, h, c = int(inf[i, 1]), int(inf[i, 2]), int(desired_channels or inf[i, 3])
        o = int(offs[i]) // out.element_size()
        views.append(out[o:o + h * w * c].view(h, w, c))
    return views


FPNGB_DECODE_BAD_CROP = 103        # decode_packed_resized_device only: the file's crop box is empty or not inside the image
FPNGB_RESIZE_ANTIALIAS = 1
FPNGB_RESIZE_ANY_PNG = 4
FPNGB_RESIZE_ALL_PNG_FORMATS = 8
FPNGB_RESIZE_NATIVE = 16
FPNGB_RESIZE_NEAREST = 32            # interpolation="nearest": F.interpolate(mode="nearest")
FPNGB_RESIZE_NEAREST_EXACT = 64      # interpolation="nearest-exact": F.interpolate(mode="nearest-exact")
FPNGB_RESIZE_INDEX = 128             # indices=True in the resized call
FPNGB_RESIZE_BICUBIC = 256           # interpolation="bicubic": F.interpolate(mode="bicubic")
FPNGB_VIEW_HFLIP = 1                 # decode_packed_views_device: view row flag, flip after the resize (torch.flip(dims=[-1]))
FPNGB_VIEW_VFLIP = 2                 # the same for rows
FPNGB_DECODE_BAD_VIEW = 106          # decode_packed_views_device only: a view row names no file, or has a bad size, offset or flag
_INTERPOLATION = {"bilinear": 0, "bicubic": FPNGB_RESIZE_BICUBIC, "nearest": FPNGB_RESIZE_NEAREST,
                  "nearest-exact": FPNGB_RESIZE_NEAREST_EXACT}


def decode_packed_resized_device(data, offsets, sizes, size, desired_channels: int, boxes=None, antialias=None, out=None, dtype=None,
                                 scale=None, bias=None, max_file_size=None, max_w=None, max_h=None, pixel_cap=None, stream=None,
                                 any_png=False, all_formats=False, native=False, interpolation="bilinear", indices=False):
    """Decode fpng files of ANY shapes packed in device memory (the layout of decode_packed_ragged_device) into one batch of a fixed
    size = (H, W): file i is cropped to boxes[i] and resized with F.interpolate's bilinear rule (align_corners=False, antialias as
    given, None meaning True) on the GPU, then stored as decode_batch_device stores its pixels (uint8, rounded half to even and clamped, or dtype with
    scale and bias).  Returns (out [n, H, W, desired_channels], info int32 [n, 6], status int32 [n]).
      * boxes: None (whole images) or an int32 CUDA tensor [n, 4] of (top, left, height, width), torchvision's resized_crop order;
      * out: any non-overlapping [n, H, W, C] view in one of the layouts of layout_strides, e.g. torch.empty(n, C, H, W,
        dtype=torch.bfloat16).permute(0, 2, 3, 1) for NCHW; by default a contiguous [n, H, W, C] tensor;
      * status[i] is decode_packed_ragged_device's code, or FPNGB_DECODE_BAD_CROP for a box that is empty or not inside the image;
        the output slice of a file whose status is not 0 is left untouched;
      * pixel_cap bounds the bytes of uint8 pixels the call decodes before resizing (align_up(w*h*desired_channels, 16) per file),
        as out's size does in decode_packed_ragged_device: files past it get FPNGB_DECODE_OUT_OF_SPACE.
    With max_file_size, max_w, max_h and pixel_cap all given, the call is stream-ordered: no host synchronisation.  Any of them
    that is None is computed by decode_packed_ragged_device's rule: one get_info_batch_device and one read-back to the host, which
    waits for the stream; pixel_cap then becomes the exact size of the decodable files.
    any_png=True decodes general PNGs too, as decode_packed_ragged_device(any_png=True) does (FPNGB_RESIZE_ANY_PNG), and
    all_formats=True (with any_png=True, else ValueError) every PNG format as there (FPNGB_RESIZE_ALL_PNG_FORMATS); the resize
    reads the uint8 values, so a 16-bit file is resized from its high bytes.
    native=True (with any_png=True, else ValueError; FPNGB_RESIZE_NATIVE) resizes every file from its 16-bit domain values (16-bit
    samples as they are, 8-bit values v as v * 257): desired_channels 1 .. 4 (1 / 2: luma and alpha, as in
    decode_packed_ragged_device(native=True)), dtype torch.uint16 stores the rounded resampled value, uint8 and the float types
    the value / 257 as above.  pixel_cap then counts bytes of the uint16 intermediate (align_up(w*h*desired_channels*2, 16) per
    file).
    interpolation="nearest" / "nearest-exact" (FPNGB_RESIZE_NEAREST / _EXACT) resizes by nearest neighbour with F.interpolate's
    rule of that mode instead: each element is, bit for bit, the element decode_packed_ragged_device with the same arguments stores
    at the source pixel, so at identity size the result is the ragged decode cropped to the box.  antialias applies to bilinear and
    bicubic only.
    interpolation="bicubic" (FPNGB_RESIZE_BICUBIC) resizes with F.interpolate's bicubic rule (align_corners=False; A = -0.75, the
    border of the box replicated) or, with antialias=True, torch's antialiased bicubic, which applies at every scale, upscaling
    included.  antialias must be given as True or False with bicubic (None raises ValueError): torch's F.interpolate defaults to
    False and torchvision's resize to True, and unlike bilinear the two bicubic rules differ at every scale, so no default would
    be right for both kinds of caller.  Bicubic overshoots: uint8 output is the rounded value clamped to 0..255 (torchvision v2's uint8 result on CUDA),
    float output keeps values below 0 and above 255 (times scale, plus bias), as torch's float result does.
    indices=True (FPNGB_RESIZE_INDEX) takes decode_packed_ragged_device's indices rule and needs a nearest mode as well; pixel_cap
    then counts align_up(w*h*element_size, 16) bytes per file."""
    out, info, status, _ = _resized_call("decode_packed_resized_device", data, offsets, sizes, size, desired_channels, boxes, None, None,
                                         antialias, out, dtype, scale, bias, max_file_size, max_w, max_h, pixel_cap, stream, any_png,
                                         all_formats, native, interpolation, indices)
    return out, info, status


def decode_packed_views_device(data, offsets, sizes, views, size, desired_channels: int, fill=None, antialias=None, out=None, dtype=None,
                               scale=None, bias=None, max_file_size=None, max_w=None, max_h=None, pixel_cap=None, stream=None,
                               any_png=False, all_formats=False, native=False, interpolation="bilinear", indices=False):
    """Decode the packed files of decode_packed_resized_device once and write any number of output images from them: a "view" here
    is one output image (not one of ragged_views' per-file tensors), a crop of a file resized to its own size, optionally flipped,
    and placed on a fixed canvas size = (H, W) holding a fill value elsewhere (fpngb_decode_packed_views_device in
    include/fpng_b200.h).  Returns (out [m, H, W, desired_channels], info int32 [n, 6], status int32 [n], view_status int32 [m]).
      * views: a contiguous int32 CUDA tensor [m, 10], 1 <= m <= 65535; row v = (file, top, left, height, width, resize_h,
        resize_w, offset_y, offset_x, flags), flags FPNGB_VIEW_HFLIP | FPNGB_VIEW_VFLIP.  View v is, bit for bit, what
        decode_packed_resized_device stores for that file with that box at size (resize_h, resize_w), then torch.flip for the
        flags, pasted at (offset_y, offset_x) (negative offsets and offsets past the canvas clip) onto a canvas of the fill.  A
        file may have any number of views, or none; resize_crop_views and letterbox_views build common tables, and flips or
        several views per file are plain torch ops on the table (views[:, 9] |= mask, torch.cat);
      * fill: None (zeros), one value or one per channel: a source value of the call, stored as the call stores one (uint8 as it
        is, float fill * scale + bias, native a 16-bit value, indices the raw id, e.g. 255 for "ignore"); 0..255, or 0..65535 in
        native calls and indices=True into uint16;
      * status[i] is decode_packed_ragged_device's code for file i (no box is checked per file); view_status[v] is
        FPNGB_DECODE_BAD_VIEW for a file outside 0..n-1, else the file's status, else FPNGB_DECODE_BAD_CROP for a box that is
        empty or not inside the image, else FPNGB_DECODE_BAD_VIEW for a resize size outside 1..2^24, an offset beyond +-2^24 or
        an unknown flag, else 0.  The output image of a view whose status is not 0 is left untouched;
      * out: any non-overlapping [m, H, W, C] view in the layouts of layout_strides (NCHW included).
    Every other argument is decode_packed_resized_device's, with the same rules: interpolation, antialias, indices, native,
    any_png, all_formats, dtype, scale and bias; pixel_cap and the bounds as there (all given: stream-ordered, no host
    synchronisation)."""
    return _resized_call("decode_packed_views_device", data, offsets, sizes, size, desired_channels, None, views, fill, antialias, out,
                         dtype, scale, bias, max_file_size, max_w, max_h, pixel_cap, stream, any_png, all_formats, native,
                         interpolation, indices)


def _resized_call(fn, data, offsets, sizes, size, desired_channels, boxes, views, fill, antialias, out, dtype, scale, bias,
                  max_file_size, max_w, max_h, pixel_cap, stream, any_png, all_formats, native, interpolation, indices):
    """The argument checks and the library call of decode_packed_resized_device (views None) and decode_packed_views_device"""
    import torch

    _all_formats_check(any_png, all_formats, fn, native)
    if interpolation not in _INTERPOLATION:
        raise ValueError(f"{fn}: interpolation {interpolation!r}: 'bilinear', 'bicubic', 'nearest' or 'nearest-exact'")
    if indices and interpolation in ("bilinear", "bicubic"):
        raise ValueError(f"{fn}: indices=True needs interpolation 'nearest' or 'nearest-exact'")
    if antialias is None:
        if interpolation == "bicubic":
            raise ValueError(f"{fn}: interpolation 'bicubic' needs antialias=True (torchvision's resize) or antialias=False "
                             "(F.interpolate's default); the two differ at every scale")
        antialias = True
    if desired_channels not in ((1, 2, 3, 4) if native else (3, 4)):
        raise ValueError(f"{fn}: desired_channels {desired_channels}: " + ("1 .. 4" if native else "3 or 4"))
    H, W = (int(v) for v in size)
    if not (1 <= H <= 1 << 24 and 1 <= W <= 1 << 24):
        raise ValueError(f"{fn}: size {tuple(size)}: each side in 1 .. 2^24")
    odt = _out_dtype(out, dtype)
    _indices_check(indices, any_png, all_formats, native, desired_channels, odt, fn)
    if native:
        fmt = _native_format(odt, scale, bias, desired_channels, fn)
    else:
        fmt = _pixel_format(odt, scale, bias, desired_channels, fn)
    if boxes is not None:
        if not isinstance(boxes, torch.Tensor) or not boxes.is_cuda or boxes.device != data.device:
            raise ValueError(f"boxes: a CUDA tensor on {data.device} is needed")
        n = sizes.shape[0]
        if boxes.dtype != torch.int32 or tuple(boxes.shape) != (n, 4) or not boxes.is_contiguous():
            raise ValueError(f"boxes: dtype {boxes.dtype}, shape {tuple(boxes.shape)}: a contiguous int32 [{n}, 4] tensor is needed")
    fill_arg = None
    if views is not None or fn == "decode_packed_views_device":
        fill_arg = _view_args(fn, views, fill, desired_channels, native and (not indices or odt == torch.uint16))
        if not views.is_cuda or data is None or views.device != data.device:
            raise ValueError(f"{fn}: views: a CUDA tensor on the device of data is needed")
    n = _packed_args(data, offsets, sizes)
    m = n if views is None else int(views.shape[0])
    shape = (m, H, W, desired_channels)
    if out is None:
        out = torch.empty(shape, dtype=odt, device=data.device)
    _check_arg(out, "out", data.device, odt, m * H * W * desired_channels, view=True)
    if max_file_size is None or max_w is None or max_h is None or pixel_cap is None:
        max_file_size, max_w, max_h, total = _ragged_bounds(data, offsets, sizes, n, desired_channels, max_file_size, max_w, max_h,
                                                             stream, odt.itemsize if indices else 2 if native else 1, any_png=any_png,
                                                             all_formats=all_formats)
        if pixel_cap is None:
            pixel_cap = total
    info = torch.empty((n, 6), dtype=torch.int32, device=data.device)
    status = torch.empty((n,), dtype=torch.int32, device=data.device)
    flags = ((FPNGB_RESIZE_ANTIALIAS if antialias and interpolation in ("bilinear", "bicubic") else 0) | (FPNGB_RESIZE_ANY_PNG if any_png else 0) |
             (FPNGB_RESIZE_ALL_PNG_FORMATS if all_formats else 0) | (FPNGB_RESIZE_NATIVE if native else 0) |
             _INTERPOLATION[interpolation] | (FPNGB_RESIZE_INDEX if indices else 0))
    head = (data.data_ptr(), data.numel(), offsets.data_ptr(), sizes.data_ptr(), n, min(int(max_file_size), 0xFFFFFFFF), int(max_w),
            int(max_h), int(pixel_cap))
    tail = (out.data_ptr(), *_layout(out, shape, (1, 2, 3, 4) if native else (3, 4)), info.data_ptr(), status.data_ptr())
    fmt_arg = None if fmt is None else C.byref(fmt)
    if views is None:
        rc = lib().fpngb_decode_packed_resized_device(*head, None if boxes is None else boxes.data_ptr(), W, H, desired_channels, flags,
                                                      fmt_arg, *tail, _stream(stream, data.device))
        view_status = None
    else:
        view_status = torch.empty((m,), dtype=torch.int32, device=data.device)
        rc = lib().fpngb_decode_packed_views_device(*head, views.data_ptr(), m, W, H, desired_channels, flags, fmt_arg, fill_arg, *tail,
                                                    view_status.data_ptr(), _stream(stream, data.device))
    check(rc, fn)
    return out, info, status, view_status


def _view_args(fn, views, fill, desired_channels, wide):
    """ValueError unless views is a contiguous int32 tensor [m, 10] with 1 <= m <= 65535 and fill None, one value or one per channel,
    each in 0..255 (0..65535 when wide: the call's source elements are uint16); returns fill as the C call takes it"""
    import torch

    if not isinstance(views, torch.Tensor) or views.dtype != torch.int32 or views.dim() != 2 or views.shape[1] != 10 or \
            not views.is_contiguous() or not 1 <= views.shape[0] <= 65535:
        what = f"dtype {views.dtype}, shape {tuple(views.shape)}" if isinstance(views, torch.Tensor) else type(views).__name__
        raise ValueError(f"{fn}: views: {what}: a contiguous int32 [m, 10] tensor with 1 <= m <= 65535 is needed")
    if fill is None:
        return None
    a = np.asarray(fill.detach().cpu().numpy() if hasattr(fill, "detach") else fill).reshape(-1)
    if a.size == 1:
        a = np.repeat(a, desired_channels)
    top = 65535 if wide else 255
    if a.size != desired_channels or not np.issubdtype(a.dtype, np.integer) or (a < 0).any() or (a > top).any():
        raise ValueError(f"{fn}: fill {fill!r}: one integer or one per channel ({desired_channels}), each in 0..{top}")
    return (C.c_uint32 * desired_channels)(*(int(v) for v in a))


def _views_table(info, rh, rw, oy, ox, h, w):
    """int32 [n, 10] rows (i, 0, 0, h, w, rh, rw, oy, ox, 0) from [n] int64 tensors"""
    import torch

    n = info.shape[0]
    i = torch.arange(n, device=info.device, dtype=torch.int64)
    z = torch.zeros_like(i)
    return torch.stack([i, z, z, h, w, rh, rw, oy, ox, z], 1).to(torch.int32).contiguous()


def resize_crop_views(info, resize, crop, max_size=None):
    """View table [n, 10] (decode_packed_views_device) of torchvision v2's Resize(resize, max_size=max_size) followed by
    CenterCrop(crop), for the files of info (get_info_batch_device's [n, 6]); use it with size = crop.  Each row is file i's whole
    image resized to (rh, rw) and placed at (oy, ox), flags 0: torch ops on the device, no host synchronisation.
      * resize: an int (the shorter side becomes resize, the longer int(resize * long / short) in float64; with max_size, when the
        longer side would pass max_size, it becomes max_size and the shorter int(max_size * short / long)) or (h, w);
      * crop: an int or (h, w).  Per axis the offset is -round((size - crop) / 2), half to even, when the crop fits and
        +(crop - size) // 2 when it does not (torchvision pads with zeros: the fill).
    Rows of files with w = h = 0 (a failed walk) hold anything: those views get the file's status first."""
    import torch

    ch, cw = (crop, crop) if isinstance(crop, int) else (int(crop[0]), int(crop[1]))
    h = info[:, 2].to(torch.int64)
    w = info[:, 1].to(torch.int64)
    if isinstance(resize, int):
        hf, wf = h.double(), w.double()
        short, long_ = torch.minimum(hf, wf), torch.maximum(hf, wf)
        new_short = torch.full_like(hf, float(resize))
        new_long = torch.floor(resize * long_ / short.clamp(min=1))
        if max_size is not None:
            over = new_long > max_size
            new_short = torch.where(over, torch.floor(max_size * new_short / new_long.clamp(min=1)), new_short)
            new_long = torch.where(over, torch.full_like(new_long, float(max_size)), new_long)
        rh = torch.where(hf <= wf, new_short, new_long).to(torch.int64)
        rw = torch.where(hf <= wf, new_long, new_short).to(torch.int64)
    else:
        if max_size is not None:
            raise ValueError("resize_crop_views: max_size applies to an int resize only (torchvision's rule)")
        rh = torch.full_like(h, int(resize[0]))
        rw = torch.full_like(w, int(resize[1]))

    def offset(size, c):
        fits = torch.round((size - c).double() / 2).to(torch.int64)     # torch.round: half to even, as Python's round
        return torch.where(size >= c, -fits, torch.div(c - size, 2, rounding_mode="floor"))

    return _views_table(info, rh, rw, offset(rh, ch), offset(rw, cw), h, w)


def letterbox_views(info, size):
    """View table [n, 10] (decode_packed_views_device) of the usual detection letterbox into a canvas size = (H, W): r = min(H / h,
    W / w) in float64, the whole image resized to rw, rh = round(w * r), round(h * r) (half to even, at least 1) and placed at
    round((canvas - resized) / 2 - 0.1) per axis, flags 0; pass the pad colour as fill.  The geometry is YOLO's; the resample is
    this library's (torch's bilinear rule with antialias as the call sets it), not OpenCV's cv2.resize, so pixels differ from an
    OpenCV pipeline.  Torch ops on the device, no host synchronisation; rows of files with w = h = 0 hold anything."""
    import torch

    H, W = (int(v) for v in size)
    h = info[:, 2].to(torch.int64)
    w = info[:, 1].to(torch.int64)
    r = torch.minimum(H / h.double().clamp(min=1), W / w.double().clamp(min=1))
    rh = torch.round(h.double() * r).clamp(min=1).to(torch.int64)
    rw = torch.round(w.double() * r).clamp(min=1).to(torch.int64)
    oy = torch.round((H - rh).double() / 2 - 0.1).to(torch.int64)
    ox = torch.round((W - rw).double() / 2 - 0.1).to(torch.int64)
    return _views_table(info, rh, rw, oy, ox, h, w)


def decode_batch_host(file_ptrs, sizes, desired_channels: int, out, out_stride: int):
    """Pipelined host-buffer batch decode (fpngb_decode_batch_host).  file_ptrs: array of host addresses (uint64), sizes:
    uint32 array, out: host buffer (numpy uint8 / pinned torch tensor) with out_stride bytes per image.
    Returns (rc, w, h, chans, status[n])."""
    n = len(sizes)
    ptrs = (C.c_void_p * n)(*[int(p) for p in file_ptrs])
    sz = np.ascontiguousarray(sizes, dtype=np.uint32)
    status = np.zeros(n, dtype=np.int32)
    w, h, c = C.c_uint32(), C.c_uint32(), C.c_uint32()
    optr = out.data_ptr() if hasattr(out, "data_ptr") else out.ctypes.data
    rc = lib().fpngb_decode_batch_host(ptrs, sz.ctypes.data_as(C.c_void_p), n, desired_channels, optr, out_stride,
                                       C.byref(w), C.byref(h), C.byref(c), status.ctypes.data_as(C.c_void_p))
    return rc, w.value, h.value, c.value, status


def decode_files(files, desired_channels: int):
    """Batch form of fpng_decode_memory (src/fpng.h:108) for a list of files (bytes-like) of ANY mix of dimensions: the C ABI decodes
    one shape per call (one kernel grid per shape), so the files are container-walked on the host, grouped by (width, height,
    channels) and every group goes through fpngb_decode_batch_host.  Returns one (status, pixels or None, w, h, chans_in_file) per
    file, in input order; status is the FPNG_DECODE_* code fpng_decode_memory would return for that file."""
    if desired_channels not in (3, 4):
        return [(FPNG_DECODE_INVALID_ARG, None, 0, 0, 0) for _ in files]
    bufs = [_u8(f) for f in files]
    results = [None] * len(bufs)
    groups = {}
    for i, a in enumerate(bufs):
        if a.size == 0:
            results[i] = (FPNG_DECODE_INVALID_ARG, None, 0, 0, 0)
            continue
        st, w, h, c, _, _ = get_info_ex(a)
        if st != FPNG_DECODE_SUCCESS:
            results[i] = (st, None, w, h, c)
        elif w * h * desired_channels > 0xFFFFFFFF:
            results[i] = (FPNG_DECODE_FAILED_DIMENSIONS_TOO_LARGE, None, w, h, c)                 # fpng.cpp:3103-3105
        else:
            groups.setdefault((w, h, c), []).append(i)
    for (w, h, c), idx in groups.items():
        need = w * h * desired_channels
        out = np.empty((len(idx), need), dtype=np.uint8)
        rc, ww, hh, cc, status = decode_batch_host([bufs[i].ctypes.data for i in idx], [bufs[i].size for i in idx], desired_channels, out, need)
        check(rc, "decode_files")
        for k, i in enumerate(idx):
            ok = int(status[k]) == FPNG_DECODE_SUCCESS
            results[i] = (int(status[k]), out[k].copy() if ok else None, w, h, c)
    return results


# ---- static-table training (reference: FPNG_TRAIN_HUFFMAN_TABLES / fpng_test -t; src/fpng.h:114-120) ----
def train_accumulate_device(images, counts=None, stream=None):
    """Adds the 16-bit scaled symbol counts of every image of a CUDA uint8 batch [n, h, w, chans] to counts[288] (uint64)."""
    import torch

    assert images.is_cuda and images.dtype == torch.uint8 and images.is_contiguous() and images.dim() == 4
    n, h, w, c = images.shape
    if counts is None:
        counts = np.zeros(288, dtype=np.uint64)
    s = _stream(stream, images.device)
    check(lib().fpngb_train_accumulate_device(images.data_ptr(), h * w * c, n, w, h, c, counts.ctypes.data_as(C.c_void_p), s), "train_accumulate_device")
    return counts


def create_dynamic_block_prefix(counts, num_chans: int):
    """src/fpng.cpp:910. Returns (prefix bytes, bit_buf, bit_buf_size, codes[288], code sizes[288])."""
    counts = np.ascontiguousarray(counts, dtype=np.uint64)
    prefix = np.zeros(4096, np.uint8); n = C.c_size_t(); bb = C.c_uint64(); bs = C.c_int()
    codes = np.zeros(288, np.uint32); sizes = np.zeros(288, np.uint8)
    check(lib().fpngb_create_dynamic_block_prefix(counts.ctypes.data_as(C.c_void_p), num_chans, prefix.ctypes.data_as(C.c_void_p), prefix.size,
                                                  C.byref(n), C.byref(bb), C.byref(bs), codes.ctypes.data_as(C.c_void_p),
                                                  sizes.ctypes.data_as(C.c_void_p)), "create_dynamic_block_prefix")
    return prefix[: n.value].tobytes(), bb.value, bs.value, codes, sizes


def set_static_table(num_chans: int, prefix: bytes = b"", bit_buf: int = 0, bit_buf_size: int = 0) -> None:
    """Install a trained 1-pass table for num_chans (empty prefix restores the built-in table)."""
    a = np.frombuffer(prefix, dtype=np.uint8) if prefix else np.zeros(1, np.uint8)
    check(lib().fpngb_set_static_table(num_chans, a.ctypes.data_as(C.c_void_p), len(prefix), bit_buf, bit_buf_size), "set_static_table")
