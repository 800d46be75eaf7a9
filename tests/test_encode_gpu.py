"""GPU parity tests of the encode hot path, through the C ABI (fpngb_encode_host / fpngb_encode_batch_device /
fpngb_encode_batch_host).  Bit-exact bar: the CUDA output must equal the oracle's bytes (which equal the reference's),
match the committed golden vectors, and round-trip through the reference decoder, lodepng and stb_image.
Mirrors the reference's own test strategy (src/fpng_test.cpp:1237-1445 round trips, 381-682 fuzz families, -u, -s)."""
import ctypes as C

import numpy as np
import pytest

import imagegen
from common import golden_vectors, sha

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1), (1, 9), (2, 2), (5, 3), (15, 2), (16, 2), (20, 1), (24, 1), (63, 3), (64, 3), (65, 3), (85, 2), (86, 2), (127, 5),
          (128, 4), (129, 6), (255, 3), (256, 3), (257, 33), (340, 5), (512, 64), (687, 41), (1000, 3), (2049, 2),
          (528, 3), (1024, 5), (1040, 2), (1920, 3), (4096, 2), (8192, 1)]   # multi-step rows on the 16-pixel-per-lane kernels


@pytest.fixture
def rows_per_warp(request):
    """Forces the scanlines-per-warp shape of the 16-pixel scan/pack kernels (large batches use 5, small ones 1; 0 = automatic)
    so that small test images exercise the pipelined multi-scanline sequence too."""
    from fpng_b200 import _lib
    _lib.lib().fpngb_debug_rows_per_warp(request.param)
    yield request.param
    _lib.lib().fpngb_debug_rows_per_warp(0)


@pytest.mark.parametrize("rows_per_warp", [5, 1, 3], indirect=True)
@pytest.mark.parametrize("kind", ["g0", "g1", "g2", "runs", "mut", "zero"])
@pytest.mark.parametrize("chans", [3, 4])
def test_encode_byte_exact_vs_oracle(gpu, oracle, kind, chans, rows_per_warp):
    for i, (w, h) in enumerate(SHAPES + [(512, 23), (1040, 11)]):
        img = imagegen.make(kind, w, h, chans, 100 + i)
        for flags in (0, gpu.FPNG_ENCODE_SLOWER, gpu.FPNG_FORCE_UNCOMPRESSED):
            ok, png = gpu.fpng_encode_image_to_memory(img, w, h, chans, flags)
            assert ok
            exp = oracle.encode(img, w, h, chans, flags)
            assert png == exp, (kind, w, h, chans, flags, rows_per_warp, len(png), len(exp))


def test_encode_matches_golden_vectors(gpu):
    for v in golden_vectors():
        img = imagegen.make(v["kind"], v["w"], v["h"], v["chans"], v["index"])
        ok, png = gpu.fpng_encode_image_to_memory(img, v["w"], v["h"], v["chans"], v["flags"])
        assert ok and len(png) == v["size"] and sha(png) == v["png_sha256"], v


def test_encode_round_trips_through_independent_decoders(gpu, ref):
    for (kind, w, h, c) in (("g1", 301, 57, 3), ("g1", 300, 57, 4), ("runs", 1024, 9, 4), ("g2", 77, 31, 3), ("g0", 640, 48, 4), ("mut", 333, 21, 3)):
        img = imagegen.make(kind, w, h, c, 5)
        for flags in (0, 1, 2):
            ok, png = gpu.fpng_encode_image_to_memory(img, w, h, c, flags)
            assert ok
            st, px, ww, hh, cc = ref.decode(png, c)                       # the reference's own decoder
            assert st == 0 and (ww, hh, cc) == (w, h, c) and np.array_equal(px, img.reshape(-1))
            err, px, ww, hh = ref.lodepng_decode(png, c)                    # checks IDAT CRC-32 and Adler-32
            assert err == 0 and np.array_equal(px, img.reshape(-1))
            comp, px, ww, hh = ref.stb_decode(png, c)
            assert comp == c and np.array_equal(px, img.reshape(-1))
            assert png == ref.encode(img, w, h, c, flags)                   # byte-exact with the reference encoder


def test_encode_round_trips_through_wuffs_and_pvpng(gpu, verifiers):
    """The harness's other two verifiers (src/fpng_test.cpp:1403-1445 wuffs, 1571-1606 pvpng) on GPU-written files; wuffs runs with
    its checksum verification ON (the harness switches it off), so it also checks the device-computed IDAT CRC-32 and Adler-32."""
    for (kind, w, h, c) in (("g1", 301, 57, 3), ("g1", 300, 57, 4), ("runs", 1024, 9, 4), ("g2", 77, 31, 3), ("g0", 640, 48, 4), ("mut", 333, 21, 3)):
        img = np.asarray(imagegen.make(kind, w, h, c, 5)).reshape(h, w, c)
        rgba = img if c == 4 else np.concatenate([img, np.full((h, w, 1), 255, np.uint8)], axis=2)
        for flags in (0, 1, 2):
            ok, png = gpu.fpng_encode_image_to_memory(img, w, h, c, flags)
            assert ok
            rc, px, ww, hh = verifiers.wuffs_decode_rgba(png, w, h)
            assert rc == 0 and (ww, hh) == (w, h) and np.array_equal(px, rgba.reshape(-1)), (kind, w, h, c, flags)
            rc, px, ww, hh, cc = verifiers.pvpng_decode(png, c, w, h)
            assert rc == 0 and (ww, hh, cc) == (w, h, c) and np.array_equal(px, img.reshape(-1)), (kind, w, h, c, flags)


def test_encode_python_zlib_and_crc(gpu):
    import struct
    import zlib
    img = imagegen.make("g1", 200, 50, 4, 9)
    ok, png = gpu.fpng_encode_image_to_memory(img, 200, 50, 4, 0)
    assert ok and png[:8] == b"\x89PNG\r\n\x1a\n"
    idat_len = struct.unpack(">I", png[50:54])[0]
    assert png[54:58] == b"IDAT" and len(png) == 58 + idat_len + 16
    raw = zlib.decompress(png[58:58 + idat_len])
    assert len(raw) == (200 * 4 + 1) * 50
    assert zlib.crc32(png[54:58 + idat_len]) == struct.unpack(">I", png[58 + idat_len:62 + idat_len])[0]


def test_encode_invalid_arguments(gpu):
    # src/fpng.cpp:1670-1680: returns false
    assert gpu.fpng_encode_image_to_memory(bytes(12), 0, 2, 3)[0] is False
    assert gpu.fpng_encode_image_to_memory(bytes(12), 2, 2, 5)[0] is False
    assert gpu.fpng_encode_image_to_memory(bytes(11), 2, 2, 3)[0] is False
    assert gpu.fpng_encode_image_to_memory(bytes(12), (1 << 24) + 1, 1, 3)[0] is False


def test_batch_device_api(gpu, oracle):
    import torch
    for (w, h, c, n, flags) in ((640, 36, 3, 5, 0), (256, 40, 4, 7, 0), (255, 17, 3, 4, 0), (130, 20, 4, 3, 1), (96, 8, 3, 3, 2)):
        imgs = np.stack([imagegen.make(["g1", "g0", "runs", "g2"][i % 4], w, h, c, i) for i in range(n)])
        t = torch.from_numpy(imgs).cuda()
        out, sizes = gpu.encode_batch_device(t, flags)
        torch.cuda.synchronize()
        sizes = sizes.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
        out = out.cpu().numpy()
        for i in range(n):
            assert bytes(out[i, : sizes[i]]) == oracle.encode(imgs[i], w, h, c, flags), (w, h, c, i, flags)


def test_batch_device_unaligned_views(gpu, oracle):
    """Images whose base address is not 16/4-byte aligned take the byte-load kernels."""
    import torch
    w, h, c, n = 37, 11, 3, 3
    imgs = np.stack([imagegen.make("g1", w, h, c, i) for i in range(n)])
    buf = torch.zeros(n * w * h * c + 1, dtype=torch.uint8, device="cuda")
    buf[1:] = torch.from_numpy(imgs.reshape(-1)).cuda()
    view = buf[1:].view(n, h, w, c)
    out, sizes = gpu.encode_batch_device(view, 0)
    torch.cuda.synchronize()
    sizes = sizes.cpu().numpy().astype(np.int64)
    out = out.cpu().numpy()
    for i in range(n):
        assert bytes(out[i, : sizes[i]]) == oracle.encode(imgs[i], w, h, c, 0)


def test_batch_host_api(gpu, oracle):
    from fpng_b200._lib import lib
    L = lib()
    w, h, c, n = 512, 300, 4, 9
    imgs = np.stack([imagegen.make(["g1", "g0", "g2"][i % 3], w, h, c, i) for i in range(n)])
    stride = gpu.max_encoded_size(w, h, c)
    out = np.zeros((n, stride), np.uint8)
    sizes = np.zeros(n, np.uint32)
    rc = L.fpngb_encode_batch_host(imgs.ctypes.data_as(C.c_void_p), w * h * c, n, w, h, c, 0, out.ctypes.data_as(C.c_void_p), stride,
                                   sizes.ctypes.data_as(C.c_void_p))
    assert rc == 0
    for i in range(n):
        assert bytes(out[i, : sizes[i]]) == oracle.encode(imgs[i], w, h, c, 0), i


def test_full_size_configs_properties(gpu, ref):
    """BASELINE.json shapes at full size: size-independent checks (decode round trip, checksum of checksums)."""
    import torch
    import zlib
    for (w, h, c, flags) in ((1920, 1080, 3, 0), (3840, 2160, 4, 0), (2048, 2048, 3, 1), (512, 512, 4, 0)):
        imgs = np.stack([imagegen.make(k, w, h, c, 3) for k in ("g1", "g0")])
        out, sizes = gpu.encode_batch_device(torch.from_numpy(imgs).cuda(), flags)
        torch.cuda.synchronize()
        sizes = sizes.cpu().numpy().astype(np.int64)
        out = out.cpu().numpy()
        for i in range(2):
            png = bytes(out[i, : sizes[i]])
            raw = zlib.decompress(png[58:-16])                      # verifies Adler-32
            assert zlib.crc32(png[54:-16]) == int.from_bytes(png[-16:-12], "big")
            assert len(raw) == (w * c + 1) * h
            st, px, *_ = ref.decode(png, c)
            assert st == 0 and np.array_equal(px, imgs[i].reshape(-1))
            assert png == ref.encode(imgs[i], w, h, c, flags)        # 1-pass and 2-pass alike (C4 = 2048^2, FPNG_ENCODE_SLOWER)


def test_checksum_utilities(gpu, oracle):
    rs = np.random.RandomState(1)
    for n in (1, 3, 4, 57, 4095, 4096, 4097, 65536, 65537, 1 << 20, (1 << 20) + 13, 5_000_001):
        d = rs.randint(0, 256, size=n, dtype=np.uint8)
        assert gpu.fpng_crc32(d) == oracle.crc32(d), n
        assert gpu.fpng_adler32(d) == oracle.adler32(d), n
        assert gpu.fpng_crc32(d, 0x12345678) == oracle.crc32(d, 0x12345678), n
        assert gpu.fpng_adler32(d, 0x00030002) == oracle.adler32(d, 0x00030002), n
    assert gpu.fpng_crc32(b"123456789") == 0xCBF43926
    assert gpu.fpng_adler32(b"Wikipedia") == 0x11E60398
    # fpng_crc32 from 4 KiB on runs idat_crc_stream_kernel over the buffer placed at device byte 54 (where "IDAT" sits in a
    # file): floor((54 + n) / 4) - 13 whole words and (54 + n) % 4 tail bytes, k whole 64 KiB CTAs for n in [65536k - 2, 65536k + 1]
    base = rs.randint(0, 256, size=(1 << 17) + 64, dtype=np.uint8)
    sizes = [4095, 4096, 4097, 200_000, 200_001, 200_002, 200_003] + [65536 * k + d for k in (1, 2) for d in range(-5, 6)]
    for n in sizes:
        for ofs in (0, 1, 2, 3):                                             # host buffers at every byte alignment
            d = base[ofs:ofs + n]
            for prev in (0, 0x12345678, 0xFFFFFFFF):
                assert gpu.fpng_crc32(d, prev) == oracle.crc32(d, prev), (n, ofs, prev)
    # chaining, with the cut on both sides of the 4 KiB switch between the host and the device routine
    d = base[:70_001]
    for cut in (4095, 4096, 4097, d.size - 4097, d.size - 4096, d.size - 4095):
        assert gpu.fpng_crc32(d[cut:], gpu.fpng_crc32(d[:cut])) == oracle.crc32(d), cut


def test_trained_rgba_table_parity(gpu, oracle):
    """Under the RGBA fixture table of tests/golden/trained_tables.json, whose one-pixel-match rule fires, RGBA 1-pass runs the
    scan and pack kernels' LIT1 instantiations: every image must equal the oracle running the same table (RGB and 2-pass keep
    their usual kernels), with one and with five scanlines per pack warp."""
    from fpng_b200 import _lib
    from test_trained_tables_cpu import load_tables
    t = load_tables()["4"]
    sizes = np.array(t["sizes"], np.uint8)
    pal = [int(v) for v in np.argsort(sizes[:256], kind="stable")[:4]]
    prefix = bytes.fromhex(t["prefix"])
    assert oracle.set_static_table(4, prefix, t["bit_buf"], t["bit_buf_size"])
    try:
        gpu.set_static_table(4, prefix, t["bit_buf"], t["bit_buf_size"])
        for rpw in (1, 5):
            _lib.lib().fpngb_debug_rows_per_warp(rpw)
            for (w, h) in ((16, 2), (512, 9), (1024, 5), (1920, 3), (4096, 2)):
                for c in (3, 4):
                    imgs = [(kind, imagegen.make(kind, w, h, c, 3)) for kind in ("g1", "g0", "runs", "g2")]
                    imgs.append(("short_runs", imagegen.short_runs(w, h, c, 5, pal)))
                    for kind, img in imgs:
                        for flags in (0, 1):
                            ok, png = gpu.fpng_encode_image_to_memory(img, w, h, c, flags)
                            assert ok and png == oracle.encode(img, w, h, c, flags), (rpw, kind, w, h, c, flags)
    finally:
        _lib.lib().fpngb_debug_rows_per_warp(0)
        gpu.set_static_table(4)
        oracle.set_static_table(4)


def test_concurrent_host_threads_and_streams(gpu, oracle):
    """Entry points are callable from several host threads (serialised internally) and on different CUDA streams."""
    import threading
    import torch
    imgs = {i: imagegen.make("g1", 320 + 16 * i, 40 + i, 3 + (i & 1), i) for i in range(8)}
    exp = {i: oracle.encode(im, im.shape[1], im.shape[0], im.shape[2], 0) for i, im in imgs.items()}
    errs = []

    def worker(i):
        for _ in range(5):
            ok, png = gpu.fpng_encode_image_to_memory(imgs[i], imgs[i].shape[1], imgs[i].shape[0], imgs[i].shape[2], 0)
            if not ok or png != exp[i]:
                errs.append(i)
            st, px, *_ = gpu.fpng_decode_memory(png, imgs[i].shape[2])
            if st != 0 or not np.array_equal(px, imgs[i].reshape(-1)):
                errs.append(100 + i)

    ts = [threading.Thread(target=worker, args=(i,)) for i in range(8)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    assert not errs
    # two streams, back-to-back batch calls sharing the workspace
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    a = torch.from_numpy(np.stack([imagegen.make("g1", 512, 64, 4, i) for i in range(6)])).cuda()
    b = torch.from_numpy(np.stack([imagegen.make("g0", 512, 64, 4, i) for i in range(6)])).cuda()
    torch.cuda.synchronize()
    outs = []
    for rep in range(4):
        oa, sa = gpu.encode_batch_device(a, 0, stream=s1.cuda_stream)
        ob, sb = gpu.encode_batch_device(b, 0, stream=s2.cuda_stream)
        outs.append((oa, sa, ob, sb))
    torch.cuda.synchronize()
    for oa, sa, ob, sb in outs:
        for t, o, s in ((a, oa, sa), (b, ob, sb)):
            sz = s.cpu().numpy().astype(np.int64)
            for i in range(6):
                assert bytes(o[i, : sz[i]].cpu().numpy()) == oracle.encode(t[i].cpu().numpy(), 512, 64, 4, 0)


def test_random_dimension_fuzz_like_reference_E(gpu, oracle):
    """The reference's `-E` fuzz (src/fpng_test.cpp:617-682): random width/height up to 8193, random 3/4 channels, uniform
    random pixels (stored-block path), verified by decoding; here additionally byte-compared with the oracle."""
    rs = np.random.RandomState(2024)
    dims = [(int(rs.randint(1, 2100)), int(rs.randint(1, 260))) for _ in range(10)] + [(8193, 3), (5, 8193), (8192, 2), (65540, 1), (21846, 4)]
    for i, (w, h) in enumerate(dims):
        c = 4 if rs.randint(0, 2) else 3
        img = rs.randint(0, 256, size=(h, w, c), dtype=np.uint8)
        ok, png = gpu.fpng_encode_image_to_memory(img, w, h, c, 0)
        assert ok and png == oracle.encode(img, w, h, c, 0), (w, h, c)
        st, px, ww, hh, cc = gpu.fpng_decode_memory(png, c)
        assert st == 0 and (ww, hh, cc) == (w, h, c) and np.array_equal(px, img.reshape(-1)), (w, h, c)
        if i % 3 == 0:   # compressible content at the same odd shapes
            img2 = imagegen.make("mut", w, h, c, i)
            for flags in (0, 1):
                ok, png = gpu.fpng_encode_image_to_memory(img2, w, h, c, flags)
                assert ok and png == oracle.encode(img2, w, h, c, flags), (w, h, c, flags)
                st, px, *_ = gpu.fpng_decode_memory(png, 7 - c)
                assert st == 0


@pytest.mark.parametrize("mode", ["fused", "two_kernel", "two_kernel_chunked", "two_kernel_file_crc", "two_kernel_file_crc_chunked"])
def test_encoder_generations_agree_with_oracle(gpu, oracle, mode):
    """The single-pass encoder (encode_fused.cu: decoupled look-back, lane-local bit strings, in-kernel CRC partials) and the
    two-kernel scan + pack encoder (default: scanline CRCs from the pack kernel; with the file-reading CRC kernel; each also cut
    into chunks with the CRC work on a side stream) must all write the reference's bytes."""
    import torch
    from fpng_b200._lib import lib
    L = lib()
    L.fpngb_debug_use_fused(1 if mode == "fused" else 0)
    L.fpngb_debug_crc_overlap(1 if mode.endswith("_chunked") else 0)
    L.fpngb_debug_pack_crc(0 if "file_crc" in mode else 1)
    try:
        # aligned and unaligned scanlines (the single-pass kernel has a staged-tile and a direct-load variant), partial units,
        # widths beyond its reach (> 4096: two-kernel encoder), one-pixel and one-row images
        shapes = [(16, 1), (16, 2), (16, 40), (32, 3), (512, 9), (528, 17), (1024, 5), (1040, 33), (1920, 8), (2048, 4), (4096, 3), (4080, 7),
                  (3840, 5), (64, 300), (1536, 11), (4112, 3), (1, 1), (1, 9), (2, 2), (5, 3), (85, 2), (86, 2), (687, 41), (513, 6), (1023, 4),
                  (2049, 3), (4095, 2), (4097, 2), (341, 25)]
        for kind in ("g1", "g0", "runs", "g2", "mut", "zero"):
            for (w, h) in shapes:
                for c in (3, 4):
                    for flags in (0, 1):
                        nimg = 17 if (w, h) == (512, 9) else 3      # >= 16 images: the chunked path with the CRC on the side stream
                        imgs = np.stack([imagegen.make(kind, w, h, c, 3 + i) for i in range(nimg)])
                        out, sizes = gpu.encode_batch_device(torch.from_numpy(imgs).cuda(), flags)
                        torch.cuda.synchronize()
                        sz = sizes.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
                        oh = out.cpu().numpy()
                        for i in range(nimg):
                            assert oh[i, : sz[i]].tobytes() == oracle.encode(imgs[i], w, h, c, flags), (mode, kind, w, h, c, flags, i)
    finally:
        L.fpngb_debug_use_fused(-1)
        L.fpngb_debug_crc_overlap(0)
        L.fpngb_debug_pack_crc(1)


def test_single_pass_encoder_many_groups(gpu, ref):
    """(single-pass encoder selected explicitly) Long look-back chains: tall images (thousands of row groups per image) and a batch mixing compressible images with
    ones that fall back to stored blocks after the single-pass kernel already wrote into their buffers."""
    import torch
    from fpng_b200._lib import lib
    lib().fpngb_debug_use_fused(1)
    try:
        _many_groups(gpu, ref)
    finally:
        lib().fpngb_debug_use_fused(-1)


def _many_groups(gpu, ref):
    import torch
    for (w, h, c) in ((512, 6000, 3), (1024, 3000, 4), (4096, 700, 4)):
        kinds = ["g1", "g2", "g0", "runs", "g2", "mut"]
        imgs = np.stack([imagegen.make(k, w, h, c, i) for i, k in enumerate(kinds)])
        for flags in (0, 1):
            out, sizes = gpu.encode_batch_device(torch.from_numpy(imgs).cuda(), flags)
            torch.cuda.synchronize()
            sz = sizes.cpu().numpy().astype(np.int64) & 0xFFFFFFFF
            oh = out.cpu().numpy()
            for i in range(len(kinds)):
                assert oh[i, : sz[i]].tobytes() == ref.encode(imgs[i], w, h, c, flags), (w, h, c, flags, kinds[i])
