"""GPU tests of encode_png_device at the edges of tests/pngenc_edges.py: stored files of three and more blocks (boundaries on a
filter byte, inside a 16-bit sample, between channels; exact multiples of 65535 bytes and one byte more), the compressed-vs-stored
tie, wide rows at every residue of the 32-pixel step, the 2^24 dimension limits, a zlib stream past 2^29 bytes (bit offsets past
2^32) and source views past 4 GiB.  Every file must equal the oracle's (oracle/png_encode_oracle.c) byte for byte;
tests/test_encode_png_edges_cpu.py shows that the oracle's files reach each construct."""
import ctypes as C
import struct
import zlib

import numpy as np
import pytest

import imagegen
import pngenc_edges as pe
from test_encode_png_gpu import GUARD, INVALID_ARG, check_against_oracle, dev, files

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def env():
    import fpng_b200
    from oracle.pngenc_oracle import PngEncodeOracle
    fpng_b200.fpng_init(0)
    return fpng_b200, PngEncodeOracle()


def need_free(gib):
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < (gib << 30):
        pytest.skip(f"needs {gib} GB of free device memory")


def crop_view(img):
    """img as an interior crop of a larger device canvas whose row pitch is an odd number of pixels"""
    h, w, c = img.shape
    W = w + (5 if (w + 5) % 2 else 6)
    canvas = np.zeros((h + 3, W, c), img.dtype)
    canvas[1:h + 1, 2:w + 2] = img
    return dev(canvas)[1:h + 1, 2:w + 2]


def planar_view(img):
    return dev(np.ascontiguousarray(img.transpose(2, 0, 1))).permute(1, 2, 0)


STORED = pe.stored_edges()


@pytest.mark.parametrize("flags", [0, pe.FORCE_UNCOMPRESSED])
def test_stored_edges_match_oracle(env, flags):
    """dense, crop (odd pitch) and planar (CHW) calls over every stored edge image; the repeated-row images through expand"""
    fp, o = env
    imgs = [e.img for e in STORED if not e.expand]
    check_against_oracle(fp, o, imgs, flags)
    views = [crop_view(i) for i in imgs]
    assert not views[0].is_contiguous()
    check_against_oracle(fp, o, imgs, flags, views=views)
    check_against_oracle(fp, o, imgs, flags, views=[planar_view(i) for i in imgs])
    rep = [e.img for e in STORED if e.expand]
    views = [dev(i[:1]).expand(i.shape[0], -1, -1) for i in rep]
    assert views[0].stride()[0] == 0
    check_against_oracle(fp, o, rep, flags, views=views)


def test_tie_edges_match_oracle(env):
    fp, o = env
    check_against_oracle(fp, o, [e.img for e in pe.tie_edges(o)])


@pytest.mark.parametrize("flags", [0, pe.FORCE_UNCOMPRESSED])
def test_wide_rows_match_oracle(env, flags):
    fp, o = env
    check_against_oracle(fp, o, [e.img for e in pe.wide_edges()], flags)


def test_dimension_limits_match_oracle(env):
    need_free(4)
    fp, o = env
    check_against_oracle(fp, o, [e.img for e in pe.limit_edges()])


def test_mixed_call_with_tall_image(env):
    """gray8 1 x 2^24, tiny images of every class and an fpng RGB image in one call: each file equals the image encoded alone"""
    need_free(4)
    fp, o = env
    rng = np.random.default_rng(9)
    tall = pe.limit_edges()[0].img
    tiny = [rng.integers(0, 3, (2 + k, 1 + 2 * k, c)).astype(dt) * (pe.top(dt) // 3) for k, (_, c, dt) in enumerate(pe.CLASSES)]
    rgb = imagegen.make("g1", 37, 11, 3, 4).reshape(11, 37, 3)
    imgs = tiny[:3] + [tall] + tiny[3:] + [rgb]
    together = files(*fp.encode_png_device([dev(i) for i in imgs]))
    for k, img in enumerate(imgs):
        assert together[k] == files(*fp.encode_png_device([dev(img)]))[0], (k, img.shape, img.dtype)
    assert together[3] == o.png_encode(tall)


def test_dimension_rejections_enqueue_nothing(env):
    """w or h of 2^24 + 1 is INVALID_ARG before anything is enqueued or written"""
    import torch
    fp, _ = env
    from fpng_b200._lib import lib
    L = lib()
    img = dev(np.zeros((4, 5, 1), np.uint8))
    out = torch.full((1 << 20,), GUARD, dtype=torch.uint8, device="cuda")
    offs = torch.full((2,), -7, dtype=torch.int64, device="cuda")
    sizes = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    before = fp.launch_count()
    for dims in ([pe.LIMIT + 1, 1, 1, 8], [1, pe.LIMIT + 1, 1, 8], [pe.LIMIT + 1, 1, 1, 16], [1, pe.LIMIT + 1, 2, 16]):
        ptrs = np.array([img.data_ptr()], np.uint64)
        d = np.array(dims, np.uint32)
        rc = L.fpngb_encode_png_ragged_device(1, ptrs.ctypes.data_as(C.c_void_p), d.ctypes.data_as(C.c_void_p), None, 0,
                                              out.data_ptr(), out.numel(), offs.data_ptr(), sizes.data_ptr(), None)
        assert rc == INVALID_ARG, dims
    torch.cuda.synchronize()
    assert fp.launch_count() == before
    assert (out == GUARD).all().item() and (offs == -7).all().item() and (sizes == -7).all().item()


def test_views_past_4gib(env):
    """gray16 rows 2^31 + 8 bytes apart (row 2 starts 4 GiB + 16 bytes past row 0) and GA16 planes 4 GiB + 2 bytes apart, in one
    call.  Row 0 of the gray16 view sits 2 GiB into its buffer, so that a row address computed in 32 bits would still read
    inside it (and give a wrong file, not a fault)."""
    import torch
    need_free(14)
    fp, o = env
    rng = np.random.default_rng(21)
    g = pe.runs_image(3, 700, 1, np.uint16, 22, run=40)
    ga = pe.runs_image(5, 90, 2, np.uint16, 23, run=30)
    g[1] = rng.integers(0, 65536, (700, 1))                           # a noise row between the runs
    row_stride, plane_stride, gbase = (1 << 31) + 8, (1 << 32) + 2, 1 << 31
    pbase = gbase + 2 * row_stride + 1408
    buf = torch.zeros((pbase + plane_stride + 2 * ga[..., 0].size + 64,), dtype=torch.uint8, device="cuda")
    for y in range(3):
        at = gbase + y * row_stride
        buf[at:at + 1400] = dev(g[y].view(np.uint8).reshape(-1))
    for j in range(2):
        at = pbase + j * plane_stride
        buf[at:at + 2 * ga[..., 0].size] = dev(np.ascontiguousarray(ga[..., j]).view(np.uint8).reshape(-1))
    u16 = buf.view(torch.uint16)
    gv = u16.as_strided((3, 700, 1), (row_stride // 2, 1, 1), gbase // 2)
    gav = u16.as_strided((5, 90, 2), (90, 1, plane_stride // 2), pbase // 2)
    for flags in (pe.FORCE_UNCOMPRESSED, 0):
        check_against_oracle(fp, o, [g, ga], flags, views=[gv, gav])
    del gv, gav, u16, buf
    torch.cuda.empty_cache()


def test_stream_past_2_29_bytes(env):
    """RGBA16 16384 x 8192 (1 GiB) written compressed (BTYPE 2) with a zlib stream over 2^29 bytes: bit offsets past 2^32.  The
    file equals the oracle's, inflates with zlib, carries a right IDAT CRC, and decodes with cv2 on the host."""
    import cv2
    import torch
    need_free(8)
    fp, o = env
    img = pe.big_rgba16()
    t = dev(img)
    out, offsets, sizes = fp.encode_png_device([t])
    got = files(out, offsets, sizes)[0]
    del t, out
    torch.cuda.empty_cache()
    zlen, btype = pe.idat_info(got)
    assert btype == 2 and zlen > (1 << 29), (zlen, btype)
    assert struct.unpack(">I", got[41 + zlen:45 + zlen])[0] == zlib.crc32(got[37:41 + zlen])
    raw = zlib.decompress(got[41:41 + zlen])
    assert len(raw) == pe.raw_size(pe.BIG_W, pe.BIG_H, 8)
    del raw
    assert got == o.png_encode(img)
    dec = cv2.imdecode(np.frombuffer(got, np.uint8), cv2.IMREAD_UNCHANGED)
    assert dec is not None and np.array_equal(dec[..., [2, 1, 0, 3]], img)
