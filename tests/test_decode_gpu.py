"""GPU parity tests of the decode hot path (fpngb_decode_host / fpngb_decode_batch_device): pixels and status codes
must equal the oracle's (== the reference decoder's) on reference-written files, including 24<->32bpp conversion,
stored-block files, 2-pass files and corrupted inputs (src/fpng_test.cpp:1237-1327, -f fuzz)."""
import numpy as np
import pytest

import imagegen
from common import golden_vectors, sha

pytestmark = pytest.mark.gpu

SHAPES = [(1, 1), (1, 9), (2, 2), (5, 3), (16, 2), (24, 1), (63, 3), (64, 3), (85, 2), (86, 2), (127, 5), (128, 4), (129, 6),
          (257, 33), (340, 5), (512, 64), (687, 41), (1000, 3), (2049, 2)]


@pytest.mark.parametrize("kind", ["g0", "g1", "g2", "runs", "mut", "zero"])
@pytest.mark.parametrize("chans", [3, 4])
def test_decode_matches_oracle(gpu, oracle, kind, chans):
    for i, (w, h) in enumerate(SHAPES):
        img = imagegen.make(kind, w, h, chans, 200 + i)
        for flags in (0, 1, 2):
            png = oracle.encode(img, w, h, chans, flags)          # byte-identical to a reference-written file
            for desired in (3, 4):
                st, px, ww, hh, cc = gpu.fpng_decode_memory(png, desired)
                est, epx, *_ = oracle.decode(png, desired)
                assert st == est == 0 and (ww, hh, cc) == (w, h, chans), (kind, w, h, chans, flags, desired, st)
                assert np.array_equal(px, epx), (kind, w, h, chans, flags, desired)


def test_decode_golden_vectors(gpu, oracle):
    for v in golden_vectors()[::3]:
        img = imagegen.make(v["kind"], v["w"], v["h"], v["chans"], v["index"])
        png = oracle.encode(img, v["w"], v["h"], v["chans"], v["flags"])
        assert sha(png) == v["png_sha256"]
        st, px, *_ = gpu.fpng_decode_memory(png, v["chans"])
        assert st == 0 and sha(px.tobytes()) == v["pixels_sha256"], v


def test_decode_reference_written_files(gpu, ref):
    for (kind, w, h, c) in (("g1", 640, 200, 3), ("g1", 640, 200, 4), ("g0", 1024, 128, 4), ("runs", 800, 60, 3), ("g2", 100, 40, 4)):
        img = imagegen.make(kind, w, h, c, 11)
        for flags in (0, 1, 2):
            png = ref.encode(img, w, h, c, flags)
            for d in (3, 4):
                st, px, *_ = gpu.fpng_decode_memory(png, d)
                rst, rpx, *_ = ref.decode(png, d)
                assert st == rst == 0 and np.array_equal(px, rpx)


def test_decode_status_codes(gpu, oracle):
    img = imagegen.make("g1", 40, 6, 3, 1)
    png = oracle.encode(img, 40, 6, 3, 0)
    assert gpu.fpng_decode_memory(png, 5)[0] == gpu.FPNG_DECODE_INVALID_ARG
    assert gpu.fpng_decode_memory(b"", 3)[0] == gpu.FPNG_DECODE_INVALID_ARG
    bad = bytearray(png); bad[0] = 0
    assert gpu.fpng_decode_memory(bytes(bad), 3)[0] == gpu.FPNG_DECODE_FAILED_NOT_PNG
    bad = bytearray(png); bad[17] ^= 1
    assert gpu.fpng_decode_memory(bytes(bad), 3)[0] == gpu.FPNG_DECODE_FAILED_HEADER_CRC32
    assert gpu.fpng_decode_memory(png[:40], 3)[0] == gpu.FPNG_DECODE_FAILED_NOT_PNG
    assert gpu.fpng_decode_memory(png[:-20], 3)[0] == gpu.FPNG_DECODE_FAILED_CHUNK_PARSING
    st, w, h, c = gpu.fpng_get_info(png)
    assert (st, w, h, c) == (0, 40, 6, 3)


def test_decode_corrupted_streams_match_oracle(gpu, oracle):
    rs = np.random.RandomState(7)
    for (kind, w, h, c, flags) in (("g1", 97, 13, 4, 0), ("g0", 200, 20, 3, 0), ("g1", 64, 16, 3, 1), ("g2", 31, 9, 4, 0)):
        img = imagegen.make(kind, w, h, c, 2)
        png = oracle.encode(img, w, h, c, flags)
        for t in range(120):
            bad = bytearray(png)
            pos = int(rs.randint(0, len(bad)))
            bad[pos] ^= 1 << int(rs.randint(0, 8))
            est, epx, *_ = oracle.decode(bytes(bad), c)
            st, px, *_ = gpu.fpng_decode_memory(bytes(bad), c)
            assert st == est, (kind, pos, st, est)
            if st == 0:
                assert np.array_equal(px, epx)


def test_decode_batch_device(gpu, oracle):
    import torch
    for (w, h, c, n, flags) in ((640, 36, 3, 5, 0), (256, 40, 4, 7, 0), (130, 20, 4, 3, 1), (96, 8, 3, 3, 2)):
        imgs = [imagegen.make(["g1", "g0", "runs", "g2"][i % 4], w, h, c, i) for i in range(n)]
        files = [oracle.encode(im, w, h, c, flags) for im in imgs]
        t, stride, sizes, ofs, lens, ww, hh, cc = gpu.pack_files_for_device(files, "cuda")
        assert (ww, hh, cc) == (w, h, c)
        for d in (3, 4):
            out, status = gpu.decode_batch_device(t, sizes, ofs, lens, w, h, c, d)
            torch.cuda.synchronize()
            assert (status.cpu().numpy() == 0).all()
            out = out.cpu().numpy()
            for i in range(n):
                assert np.array_equal(out[i].reshape(-1), oracle.decode(files[i], d)[1]), (w, h, c, i, d)


def test_encode_decode_round_trip_full_size(gpu):
    """BASELINE.json shapes at full size: GPU encode -> GPU decode returns the input pixels (size-independent property)."""
    import torch
    for (w, h, c, flags) in ((1920, 1080, 3, 0), (3840, 2160, 4, 0), (2048, 2048, 3, 1)):
        imgs = np.stack([imagegen.make(k, w, h, c, 4) for k in ("g1", "g0", "g2")])
        dev = torch.from_numpy(imgs).cuda()
        out, sizes = gpu.encode_batch_device(dev, flags)
        torch.cuda.synchronize()
        sizes = sizes.cpu().numpy().astype(np.int64)
        files = [bytes(out[i, : sizes[i]].cpu().numpy()) for i in range(3)]
        t, stride, fs, ofs, lens, ww, hh, cc = gpu.pack_files_for_device(files, "cuda")
        px, status = gpu.decode_batch_device(t, fs, ofs, lens, w, h, c, c)
        torch.cuda.synchronize()
        assert (status.cpu().numpy() == 0).all()
        assert torch.equal(px, dev)


def test_decode_batch_host(gpu, oracle):
    """fpngb_decode_batch_host: pipelined host batch; bad files keep their container status and are skipped."""
    w, h, c, n = 300, 40, 3, 11
    imgs = [imagegen.make(["g1", "g0", "g2", "runs"][i % 4], w, h, c, i) for i in range(n)]
    files = [np.frombuffer(oracle.encode(im, w, h, c, i % 3), dtype=np.uint8).copy() for i, im in enumerate(imgs)]
    files[4] = files[4].copy(); files[4][0] = 0                      # not a PNG
    files[7] = files[7].copy(); files[7][90] ^= 0x10                 # corrupt stream -> NOT_FPNG (or still valid: compare with oracle)
    for d in (3, 4):
        out = np.zeros((n, w * h * d), np.uint8)
        rc, ww, hh, cc, status = gpu.decode_batch_host([f.ctypes.data for f in files], [f.size for f in files], d, out, w * h * d)
        assert rc == 0 and (ww, hh, cc) == (w, h, c)
        for i in range(n):
            est, epx, *_ = oracle.decode(files[i].tobytes(), d)
            assert status[i] == est, (i, status[i], est)
            if est == 0:
                assert np.array_equal(out[i], epx), i


def test_decode_write_pass_matches_oracle(gpu, oracle):
    """The write pass (decode_write_kernel, one thread per subsequence) must give the oracle's pixels and statuses, on clean and on
    corrupted streams; the large cases cross many scanlines / CTAs and mix matches into literal runs."""
    rs = np.random.RandomState(3)
    cases = []
    for (kind, w, h, c, flags) in (("g1", 700, 200, 3, 0), ("g1", 512, 160, 4, 0), ("mut", 1000, 120, 3, 1), ("runs", 640, 200, 4, 0),
                                    ("g0", 1600, 300, 3, 0), ("g1", 3, 3000, 4, 0), ("g1", 61, 600, 3, 1), ("zero", 900, 300, 4, 0)):
        img = imagegen.make(kind, w, h, c, 5)
        png = oracle.encode(img, w, h, c, flags)
        cases.append((png, c))
        for t in range(3):                                   # corrupted copies: statuses (and pixels when still valid) must match too
            bad = bytearray(png); pos = int(rs.randint(60, len(bad))); bad[pos] ^= 1 << int(rs.randint(0, 8))
            cases.append((bytes(bad), c))
    expect = [(oracle.decode(png, 3), oracle.decode(png, 4)) for png, c in cases]
    for (png, c), (e3, e4) in zip(cases, expect):
        for d, e in ((3, e3), (4, e4)):
            st, px, *_ = gpu.fpng_decode_memory(png, d)
            assert st == e[0], (len(png), d, st, e[0])
            if st == 0:
                assert np.array_equal(px, e[1]), (len(png), d)
